"""CPU tests of the host side: the C-ABI library loads and exports every declared symbol, fails loudly without a GPU,
the host zkey reader produces the reference's structures, and the synthetic setup is a valid Groth16 key."""
import os
import re

import numpy as np
import pytest

from oracle import cref as c
from oracle import pyref as o
from proof_model import CpuFixedBase

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_library_exports_every_declared_symbol():
    from circom_compat_b200 import _native as N
    hdr = open(os.path.join(ROOT, 'include', 'b2groth.h')).read()
    declared = set(re.findall(r'B2G_API\s+[\w\s\*]*?\b(b2g_\w+)\s*\(', hdr))
    assert len(declared) >= 20
    L = N.lib()
    for name in declared:
        assert hasattr(L, name), name
    assert declared == set(N.EXPORTS)
    assert L.b2g_version() == 1


@pytest.mark.skipif(_has_cuda(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from circom_compat_b200 import Context, B2gError
    with pytest.raises(B2gError) as e:
        Context(0)
    assert e.value.code == -3


def test_read_zkey_matches_oracle_reader(test_zkey_bytes, complex_zkey_bytes):
    from circom_compat_b200 import read_zkey
    for data in (test_zkey_bytes, complex_zkey_bytes):
        pk, cm = read_zkey(data)
        za = c.zkey_arrays(data)
        assert (pk.n_vars, pk.n_public, pk.domain_size) == (za['n_vars'], za['n_public'], za['domain_size'])
        assert cm.num_constraints == za['num_constraints'] and cm.num_instance_variables == za['n_public'] + 1
        assert cm.num_witness_variables == za['n_vars'] - za['n_public'] - 1 and cm.c_num_non_zero == 0
        for name in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query'):
            assert np.array_equal(getattr(pk, name), za[name]), name
        for i in range(3):
            assert np.array_equal(cm.a[i], za['a_csr'][i]) and np.array_equal(cm.b[i], za['b_csr'][i])
        assert cm.a_num_non_zero == len(za['a_csr'][1]) and cm.b_num_non_zero == len(za['b_csr'][1])


def test_read_zkey_rejects_garbage():
    from circom_compat_b200 import read_zkey
    with pytest.raises(ValueError):
        read_zkey(b'r1cs' + bytes(64))


def test_montgomery_helpers_roundtrip():
    from circom_compat_b200 import fr_to_mont, fr_from_mont
    vals = [0, 1, 33, o.R_MOD - 1, 12345678901234567890123456789]
    m = fr_to_mont(vals)
    assert fr_from_mont(m) == vals
    assert np.array_equal(m, c.fr_to_mont(c.ints_to_limbs(vals)))


@pytest.mark.parametrize('kind', ['chain', 'circomlike'])
def test_synthetic_setup_is_a_valid_groth16_key(kind, tmp_path):
    from circom_compat_b200 import synth, read_zkey, fr_to_mont, fr_from_mont
    if kind == 'chain':
        circ = synth.chain_circuit(64); w = synth.chain_witness(64)
    else:
        circ, w = synth.circomlike_circuit(9)
    pk, td = synth.setup(CpuFixedBase(), circ)
    assert td.h_t == o.h_query_scalars(circ.domain_size - 1, td.tau, pow(td.delta, -1, o.R_MOD))   # qap.rs:90-105 literally
    path = str(tmp_path / 'syn.zkey')
    synth.write_zkey(path, pk, circ)
    data = open(path, 'rb').read()
    za = c.zkey_arrays(data)
    r, s = 0x1234567890abcdef, 0xfedcba0987654321
    pb, h = c.prove(za, r, s, fr_to_mont(w), want_h=True)
    v = [int.from_bytes(pb[i:i + 32], 'little') for i in range(0, 256, 32)]
    proof = ((v[0], v[1]), ((v[2], v[3]), (v[4], v[5])), (v[6], v[7]))
    z = o.read_zkey(data)
    assert o.verify(z, w[1:circ.num_inputs], proof)
    da, db, dc = synth.expected_proof_dlogs(td, w, fr_from_mont(h), r, s, circ.num_inputs)
    assert o.G1.mul(o.G1_GEN, da) == proof[0] and o.G2.mul(o.G2_GEN, db) == proof[1] and o.G1.mul(o.G1_GEN, dc) == proof[2]
    # the h-free closed form (H term = (a(tau) b(tau) - c(tau)) / delta from the matrix rows): same discrete logs, and it
    # moves when the witness breaks a constraint while the h-based form follows whatever h it is given
    assert synth.expected_proof_dlogs_independent(td, circ, w, r, s) == (da, db, dc)
    wbad = list(w); wbad[5] = (wbad[5] + 1) % o.R_MOD
    hbad = fr_from_mont(c.witness_map(circ.num_constraints, circ.num_inputs, circ.n_vars, circ.matrices().a, circ.matrices().b, fr_to_mont(wbad)))
    assert synth.expected_proof_dlogs_independent(td, circ, wbad, r, s) == synth.expected_proof_dlogs(td, wbad, hbad, r, s, circ.num_inputs)
    assert synth.expected_proof_dlogs_independent(td, circ, wbad, r, s) != synth.expected_proof_dlogs(td, wbad, fr_from_mont(h), r, s, circ.num_inputs)
    pk2, cm2 = read_zkey(data)
    assert pk2.n_vars == circ.n_vars and cm2.num_constraints == circ.num_constraints


# ------------------------------------------------------------------------------------------------ C++ host mirror
HOST_BIN = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')


def _fnv(data: bytes, h: int = 1469598103934665603) -> int:
    for b in data:
        h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


@pytest.mark.parametrize('name', ['test.zkey', 'complex-circuit-10000-10000.zkey'])
def test_cpp_read_zkey_matches_python_reader(name):
    """ark_circom::read_zkey (circom_compat_b200/host/ark_circom_b200.hpp) vs the Python reader and the oracle's."""
    import subprocess
    from circom_compat_b200 import read_zkey
    path = os.path.join(ROOT, 'tests', 'golden', name)
    out = subprocess.check_output([HOST_BIN, '--parse-only', path], text=True)
    kv = dict(re.findall(r'(\w+)=(\w+)', out))
    pk, cm = read_zkey(path)
    assert (int(kv['n_vars']), int(kv['n_public']), int(kv['domain'])) == (pk.n_vars, pk.n_public, pk.domain_size)
    assert (int(kv['num_constraints']), int(kv['num_instance']), int(kv['num_witness'])) == (cm.num_constraints, cm.num_instance_variables, cm.num_witness_variables)
    assert (int(kv['a_nnz']), int(kv['b_nnz'])) == (cm.a_num_non_zero, cm.b_num_non_zero)
    for key, arr in (('a', pk.a_query), ('b1', pk.b_g1_query), ('b2', pk.b_g2_query), ('l', pk.l_query), ('h', pk.h_query), ('alpha', pk.alpha_g1)):
        if arr.size * 8 < 2_000_000:
            assert int(kv[key], 16) == _fnv(np.ascontiguousarray(arr).tobytes()), key
    if cm.a_num_non_zero < 1000:
        h = 1469598103934665603
        for rowptr, col, val in (cm.a, cm.b):
            for k in range(len(col)):
                h = _fnv(val[k].tobytes(), h); h = _fnv(int(col[k]).to_bytes(4, 'little'), h)
        assert int(kv['coefs'], 16) == h


def test_fr_rand_limb_rule():
    # SURVEY.md App. C.5: limbs from next_u64 (limb 0 first), top two bits cleared, reject >= r, limbs ARE the Montgomery residue
    from circom_compat_b200.groth16 import fr_rand

    class Stream:
        def __init__(self, words): self.words = list(words)
        def next_u64(self): return self.words.pop(0)
    R = 1 << 256
    top = o.R_MOD >> 192                                     # limb 3 of r: a draw whose limb 3 exceeds it is rejected
    rejected = [0, 0, 0, (top + 1) | (3 << 62)]              # the two flag bits are cleared first, the rest is still >= r
    accepted = [5, 6, 7, 8 | (1 << 63)]
    st = Stream(rejected + accepted + [1, 2, 3, 4])
    v = fr_rand(st)
    assert v == (5 + (6 << 64) + (7 << 128) + (8 << 192)) * pow(R, -1, o.R_MOD) % o.R_MOD
    assert len(st.words) == 4
    import random
    assert 0 <= fr_rand(random.Random(1)) < o.R_MOD


# ------------------------------------------------------------------------------------------------ product-side verifier
def test_product_verifiers_python_and_cpp(golden, test_zkey_bytes):
    """Groth16.process_vk / verify_with_processed_vk / verify (src/zkey.rs:868-870, tests/groth16.rs:33-35) in both host
    mirrors, on the golden proofs: accept, reject a wrong public input (tests/groth16.rs:42-74), reject a tampered proof,
    MalformedVerifyingKey on an input-count mismatch; must agree with the oracle's independently built pairing."""
    import subprocess
    from circom_compat_b200 import Groth16, Proof, read_zkey, MalformedVerifyingKey, verifier
    pk, cm = read_zkey(test_zkey_bytes)
    z = o.read_zkey(test_zkey_bytes)
    pvk = Groth16.process_vk(pk)
    zk = os.path.join(ROOT, 'tests', 'golden', 'test.zkey')
    for case in golden['test_zkey']['proofs']:
        p = Proof(bytes.fromhex(case['proof_hex']))
        assert Groth16.verify_with_processed_vk(pvk, [33], p) and o.verify(z, [33], (p.a, p.b, p.c))
        assert not Groth16.verify_with_processed_vk(pvk, [34], p)
        out = subprocess.check_output([HOST_BIN, '--verify', zk, case['proof_hex'], '33'], text=True) + \
            subprocess.check_output([HOST_BIN, '--verify', zk, case['proof_hex'], '34'], text=True)
        assert out.split() == ['verified=1', 'verified=0']
    p = Proof(bytes.fromhex(golden['test_zkey']['proofs'][0]['proof_hex']))
    assert Groth16.verify(pk, [33], p)
    # tampered proofs: C replaced by A (on the curve, wrong), and a coordinate bit flip (off the curve)
    swapped = Proof(p.data[:192] + p.data[:64])
    assert not Groth16.verify_with_processed_vk(pvk, [33], swapped) and not o.verify(z, [33], (swapped.a, swapped.b, swapped.c))
    flipped = bytearray(p.data); flipped[0] ^= 1
    assert not Groth16.verify_with_processed_vk(pvk, [33], Proof(bytes(flipped)))
    assert 'verified=0' in subprocess.check_output([HOST_BIN, '--verify', zk, swapped.data.hex(), '33'], text=True)
    with pytest.raises(MalformedVerifyingKey):
        Groth16.verify_with_processed_vk(pvk, [33, 1], p)
    r = subprocess.run([HOST_BIN, '--verify', zk, p.data.hex()], capture_output=True, text=True)
    assert r.returncode == 1 and 'MalformedVerifyingKey' in r.stderr
    # pairing sanity on the product's tower arithmetic: bilinear, non-degenerate, order r
    e = verifier.pairing(z.alpha_g1, z.beta_g2)
    assert verifier.pairing(verifier.g1_mul(z.alpha_g1, 5), z.beta_g2) == verifier.f12_pow(e, 5)
    assert e != verifier.F12_ONE and verifier.f12_pow(e, o.R_MOD) == verifier.F12_ONE


def test_product_verifier_degenerate_points(test_zkey_bytes):
    """Points at infinity in a proof: e(inf, Q) = e(P, inf) = 1 (arkworks' multi_miller_loop skips them); such a proof only
    verifies if the remaining equation holds, which it does not for a real key; both mirrors agree with the oracle."""
    import subprocess
    from circom_compat_b200 import Groth16, Proof, read_zkey, verifier
    pk, _ = read_zkey(test_zkey_bytes)
    z = o.read_zkey(test_zkey_bytes)
    pvk = Groth16.process_vk(pk)
    zero = Proof(bytes(256))
    assert not Groth16.verify_with_processed_vk(pvk, [33], zero)
    assert not o.verify(z, [33], (None, None, None))
    out = subprocess.check_output([HOST_BIN, '--verify', os.path.join(ROOT, 'tests', 'golden', 'test.zkey'), zero.data.hex(), '33'], text=True)
    assert 'verified=0' in out
    # pairing with infinity is the identity of GT
    assert verifier.pairing(None, z.beta_g2) == verifier.F12_ONE and verifier.pairing(z.alpha_g1, None) == verifier.F12_ONE
    # e(-P, Q) * e(P, Q) = 1
    e1 = verifier.miller_loop([(z.alpha_g1, z.beta_g2), (verifier.g1_neg(z.alpha_g1), z.beta_g2)])
    assert verifier.final_exponentiation(e1) == verifier.F12_ONE


def test_product_verifier_reference_bench_key(golden, complex_zkey_bytes):
    # benches/groth16.rs:63-66: the proof of the 10 000-constraint chain verifies with inputs = full_assignment[1..num_inputs]
    from circom_compat_b200 import Groth16, Proof, read_zkey
    pk, cm = read_zkey(complex_zkey_bytes)
    g = golden['complex_zkey']
    w = o.chain_witness(pk.n_vars, g['a'])
    p = Proof(bytes.fromhex(g['proof_hex']))
    assert Groth16.verify(pk, w[1:cm.num_instance_variables], p)
    assert not Groth16.verify(pk, [(w[1] + 1) % o.R_MOD], p)


# ------------------------------------------------------------------------------------------------ output formats
def test_proof_formats(golden, test_zkey_bytes):
    """Ethereum tuples (src/ethereum.rs) and ark-serialize encodings of a golden proof; the compressed form must
    decompress (oracle, independent sqrt) back to the same points."""
    from circom_compat_b200 import Proof, read_zkey
    from circom_compat_b200 import ethereum as eth
    case = golden['test_zkey']['proofs'][0]
    p = Proof(bytes.fromhex(case['proof_hex']))
    ep = eth.Proof.from_proof(p)
    a, b, c_ = ep.as_tuple()
    assert a == p.a and c_ == p.c
    assert b == ([p.b[0][1], p.b[0][0]], [p.b[1][1], p.b[1][0]])          # c1 first (ethereum.rs:82-86)
    assert len(ep.calldata()) == 256 and int.from_bytes(ep.calldata()[:32], 'big') == p.a[0]
    comp = eth.serialize_compressed(ep)
    assert len(comp) == 128
    assert o.decompress_proof(comp) == (p.a, p.b, p.c)
    unc = eth.serialize_uncompressed(ep)
    # ark-serialize Compress::No = x || y.serialize_with_flags(to_flags()): the YIsNegative bit (0x80) is set on the last byte
    # of y (y.c1 for G2) whenever y > -y, so the bytes equal the ABI's raw coordinates only after masking the flag bits
    assert len(unc) == 256
    raw = bytearray(unc)
    for last, neg in ((63, p.a[1] > o.Q_MOD - p.a[1]), (191, (p.b[1][1], p.b[1][0]) > ((o.Q_MOD - p.b[1][1]) % o.Q_MOD, (o.Q_MOD - p.b[1][0]) % o.Q_MOD)),
                      (255, p.c[1] > o.Q_MOD - p.c[1])):
        assert (raw[last] & 0xC0) == (0x80 if neg else 0), last
        raw[last] &= 0x3F
    assert bytes(raw) == p.data
    # the flag agrees with the compressed form's (same to_flags() value on x there)
    assert (unc[63] & 0x80) == (comp[31] & 0x80) and (unc[191] & 0x80) == (comp[95] & 0x80) and (unc[255] & 0x80) == (comp[127] & 0x80)
    inf = eth.Proof(eth.G1(0, 0), ep.b, ep.c)
    assert eth.serialize_compressed(inf)[31] == 0x40 and eth.serialize_uncompressed(inf)[63] == 0x40
    pk, _ = read_zkey(test_zkey_bytes)
    vk = eth.VerifyingKey.from_proving_key(pk)
    z = o.read_zkey(test_zkey_bytes)
    t = vk.as_tuple()
    assert t[0] == z.alpha_g1 and t[1] == ([z.beta_g2[0][1], z.beta_g2[0][0]], [z.beta_g2[1][1], z.beta_g2[1][0]])
    assert t[4] == [tuple(pt) for pt in z.ic]
    assert eth.inputs([33]) == [33]


# ------------------------------------------------------------------------------------------------ R1CS route (host readers)
R1CS_SAMPLE_HEX = """72316373 01000000 03000000 01000000 40000000 00000000 20000000
 010000f0 93f5e143 9170b979 48e83328 5d588181 b64550b8 29a031e1 724e6430 07000000 01000000 02000000 03000000 e8030000 00000000 03000000
 02000000 88020000 00000000
 02000000 05000000 03000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 06000000 08000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 00000000 02000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 02000000 14000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 0C000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 02000000 00000000 05000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 02000000 07000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 01000000 04000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 04000000 08000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 05000000 03000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 02000000 03000000 2C000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 06000000 06000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 00000000
 01000000 06000000 04000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 00000000 06000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 02000000 0B000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 05000000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 01000000 06000000 58020000 00000000 00000000 00000000 00000000 00000000 00000000 00000000
 03000000 38000000 00000000
 00000000 00000000 03000000 00000000 0a000000 00000000 0b000000 00000000 0c000000 00000000 0f000000 00000000 44010000 00000000"""


def test_r1cs_reader_reference_sample():
    # the iden3-spec sample and the assertions of /root/reference/src/circom/r1cs_reader.rs:257-338
    from circom_compat_b200 import R1CSFile
    f = R1CSFile.new(bytes.fromhex(R1CS_SAMPLE_HEX.replace('\n', '').replace(' ', '')))
    h = f.header
    assert (f.version, h.field_size, h.n_wires, h.n_pub_out, h.n_pub_in, h.n_prv_in, h.n_labels, h.n_constraints) == (1, 32, 7, 1, 2, 3, 0x03e8, 3)
    assert len(f.constraints) == 3 and len(f.constraints[0][0]) == 2
    assert f.constraints[0][0][0] == (5, 3) and f.constraints[2][1][0] == (0, 6) and len(f.constraints[1][2]) == 0
    assert len(f.wire_mapping) == 7 and f.wire_mapping[1] == 3


def test_r1cs_and_wtns_fixtures():
    from circom_compat_b200 import R1CSFile, R1CS, read_wtns
    from circom_compat_b200.r1cs import SerializationError
    data = open(os.path.join(ROOT, 'tests', 'golden', 'circuit2.r1cs'), 'rb').read()
    r = R1CS.from_file(R1CSFile.new(data))
    ni, nw, cons = o.read_r1cs(data)
    assert (r.num_inputs, r.num_variables, len(r.constraints)) == (ni, nw, len(cons)) == (2, 132, 131)
    assert all([(v, w) for w, v in mine[k]] == ref[k] for mine, ref in zip(r.constraints, cons) for k in range(3))
    w = read_wtns(open(os.path.join(ROOT, 'tests', 'golden', 'circuit2_witness.wtns'), 'rb').read())
    assert len(w) == 132 and w[:4] == [1, 33, 3, 11]
    assert all((sum(v * w[i] for i, v in c_[0]) * sum(v * w[i] for i, v in c_[1]) - sum(v * w[i] for i, v in c_[2])) % o.R_MOD == 0 for c_ in r.constraints)
    with pytest.raises(SerializationError):
        R1CSFile.new(b'zkey' + data[4:])
    circ = r.to_circuit()
    cm = circ.matrices(with_c=True)
    assert cm.c is not None and cm.num_constraints == 131 and cm.num_instance_variables == 2


def test_libsnark_oracles_agree_and_satisfy_qap_identity():
    from circom_compat_b200 import R1CSFile, R1CS, read_wtns, fr_to_mont
    data = open(os.path.join(ROOT, 'tests', 'golden', 'circuit2.r1cs'), 'rb').read()
    r = R1CS.from_file(R1CSFile.new(data))
    w = read_wtns(open(os.path.join(ROOT, 'tests', 'golden', 'circuit2_witness.wtns'), 'rb').read())
    ni, nw, cons = o.read_r1cs(data)
    A = [c_[0] for c_ in cons]; B = [c_[1] for c_ in cons]; Cm = [c_[2] for c_ in cons]
    h = o.libsnark_witness_map_from_matrices(A, B, Cm, ni, len(cons), w)
    assert len(h) == 256 and h[-1] == 0
    cm = r.to_circuit().matrices(with_c=True)
    hc = c.witness_map_libsnark(cm.num_constraints, cm.num_instance_variables, cm.a, cm.b, cm.c, fr_to_mont(w))
    assert c.limbs_to_ints(c.fr_from_mont(hc)) == h


def test_builder_api_surface():
    """CircomConfig / CircomBuilder / CircomCircuit flow of /root/reference/tests/groth16.rs:11-41 (witness from a callable
    standing in for the WASM calculator) and :106-119 (witness generation only)."""
    from circom_compat_b200 import CircomConfig, CircomBuilder
    g = os.path.join(ROOT, 'tests', 'golden')

    def mycircuit_calculator(inputs):                      # test-vectors/mycircuit.circom: c <== a * b
        a, b = inputs['a'][0], inputs['b'][0]
        return [1, a * b, a, b]
    cfg = CircomConfig.new(mycircuit_calculator, os.path.join(g, 'mycircuit.r1cs'))
    builder = CircomBuilder.new(cfg)
    builder.push_input('a', 3)
    builder.push_input('b', 11)
    circom = builder.setup()
    assert circom.witness is None and circom.get_public_inputs() is None and circom.r1cs.wire_mapping is None
    circom = builder.build()
    assert circom.witness == [1, 33, 3, 11] and circom.get_public_inputs() == [33]
    bad = CircomBuilder.new(CircomConfig.new(lambda inputs: [1, 34, 3, 11], os.path.join(g, 'mycircuit.r1cs')))
    with pytest.raises(ValueError):
        bad.build()
    # .wtns file as the witness source (circuit2, 131 constraints: tests/groth16.rs:75-105)
    c2 = CircomBuilder.new(CircomConfig.new(os.path.join(g, 'circuit2_witness.wtns'), os.path.join(g, 'circuit2.r1cs'))).build()
    assert len(c2.witness) == 132 and c2.get_public_inputs() == [33]
    circ = c2.to_circuit()
    assert circ.num_constraints == 131 and circ.num_inputs == 2


# ------------------------------------------------------------------------------------------------ malformed inputs
def test_truncated_and_corrupt_files_fail_cleanly(tmp_path, test_zkey_bytes):
    """A malformed .zkey / .r1cs / .wtns must raise (Python) or exit with an error message (C++ reader), never crash:
    the reference returns SerializationError for these (src/zkey.rs:43, r1cs_reader.rs:13)."""
    import subprocess
    from circom_compat_b200 import read_zkey, R1CSFile, read_wtns
    g = os.path.join(ROOT, 'tests', 'golden')
    r1cs = open(os.path.join(g, 'mycircuit.r1cs'), 'rb').read()
    wtns = open(os.path.join(g, 'circuit2_witness.wtns'), 'rb').read()
    for cut in (3, 11, 40, 700, len(test_zkey_bytes) - 200):          # the last 104 bytes are the unread contributions section
        with pytest.raises(Exception):
            read_zkey(test_zkey_bytes[:cut])
        f = tmp_path / ('t%d.zkey' % cut)
        f.write_bytes(test_zkey_bytes[:cut])
        r = subprocess.run([HOST_BIN, '--parse-only', str(f)], capture_output=True, text=True, timeout=30)
        assert r.returncode == 1 and 'error:' in r.stderr, (cut, r.returncode, r.stderr)
    bad = bytearray(test_zkey_bytes); bad[0:4] = b'r1cs'
    with pytest.raises(ValueError):
        read_zkey(bytes(bad))
    wrong_curve = bytearray(test_zkey_bytes)
    from circom_compat_b200.zkey import _sections
    wrong_curve[_sections(test_zkey_bytes)[2][0] + 4] ^= 1               # first byte of q in the header section
    with pytest.raises(ValueError):
        read_zkey(bytes(wrong_curve))
    for cut in (2, 20, 100, len(r1cs) - 5):
        with pytest.raises(Exception):
            R1CSFile.new(r1cs[:cut])
    for cut in (2, 30, 60):
        with pytest.raises(Exception):
            read_wtns(wtns[:cut])


def test_ntt8_index_model():
    """The register/shared-memory schedule of ntt_pass8_kernel, modelled on the CPU (tools/ntt8_model.py): forward transform ==
    DFT definition, inverse round trip, and the fused evaluations-on-H -> evaluations-on-gH chain, for one-pass, two-pass,
    three-pass and 2-D-tile schedules (small tiles stand in for the 1024/2048-element ones)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('ntt8_model', os.path.join(os.path.dirname(__file__), '..', 'tools', 'ntt8_model.py'))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    for log_n, tlmax, maxk in [(3, 3, None), (5, 5, None), (7, 7, None), (7, 4, None), (8, 4, None), (9, 5, None), (10, 4, None), (9, 5, 2), (10, 6, 3), (11, 6, None),
                              (10, 10, None), (11, 11, None), (12, 10, None), (13, 10, 7)]:   # the real 1024- and 2048-element tiles
        m.check(log_n, tlmax, maxk)


def test_ethereum_conversions_round_trip(golden, test_zkey_bytes):
    """The reference's own conversion tests (src/ethereum.rs:195-279: convert_fq, convert_fr, convert_g1, convert_g2, convert_vk,
    convert_proof) on the Python mirror, plus the tests/solidity.rs flow with the host verifier standing in for the contract:
    proof and verifying key go to Ethereum tuples (big-endian U256 words, G2 with c1 first) and come back unchanged and valid."""
    import random
    from circom_compat_b200 import Proof, read_zkey, verifier
    from circom_compat_b200 import ethereum as eth
    from circom_compat_b200.zkey import R_MOD
    rng = random.Random(0xE7)
    # convert_fq / convert_fr: field element -> U256 -> field element -> U256
    for el, mod in ((2, o.Q_MOD), (2, R_MOD), (o.Q_MOD - 1, o.Q_MOD), (R_MOD - 1, R_MOD), (rng.randrange(R_MOD), R_MOD)):
        w = eth.point_to_u256(el, mod)
        assert len(w) == 32 and int.from_bytes(w, 'big') == el
        el3 = eth.u256_to_point(w, mod)
        assert el3 == el and eth.point_to_u256(el3, mod) == w
    with pytest.raises(ValueError):
        eth.u256_to_point(o.Q_MOD.to_bytes(32, 'big'))                  # F::from_bigint(..).expect(..) panics in the reference
    # convert_g1 / convert_g2 (random points, and infinity <-> (0, 0))
    g1s = [o.G1.mul(o.G1_GEN, rng.randrange(1, R_MOD)) for _ in range(4)] + [None]
    g2s = [o.G2.mul(o.G2_GEN, rng.randrange(1, R_MOD)) for _ in range(3)] + [None]
    for el in g1s:
        el2 = eth.G1.from_affine(el); el3 = el2.to_affine(); el4 = eth.G1.from_affine(el3)
        assert el3 == el and el4 == el2 and eth.G1.from_tuple(el2.as_tuple()) == el2
    for el in g2s:
        el2 = eth.G2.from_affine(el); el3 = el2.to_affine(); el4 = eth.G2.from_affine(el3)
        assert el3 == el and el4 == el2 and eth.G2.from_tuple(el2.as_tuple()) == el2
        if el is not None:
            assert el2.as_tuple()[0] == [el[0][1], el[0][0]]            # c1 first on the wire (ethereum.rs:82-86)
    # convert_vk
    vk = verifier.VerifyingKey(g1s[0], g2s[0], g2s[1], g2s[2], [g1s[1], g1s[2], g1s[3]])
    assert eth.VerifyingKey.from_verifying_key(vk).to_verifying_key() == vk
    assert eth.VerifyingKey.from_tuple(eth.VerifyingKey.from_verifying_key(vk).as_tuple()).to_verifying_key() == vk
    # convert_proof, on a real proof
    case = golden['test_zkey']['proofs'][0]
    p = Proof(bytes.fromhex(case['proof_hex']))
    p2 = eth.Proof.from_proof(p)
    assert p2.to_proof().data == p.data
    assert eth.Proof.from_tuple(p2.as_tuple()) == p2
    # tests/solidity.rs:46-53 check_proof(proof, vk, inputs): everything through the Ethereum types, verified on the host
    pk, _ = read_zkey(test_zkey_bytes)
    vk_wire = eth.VerifyingKey.from_verifying_key(verifier.VerifyingKey.from_proving_key(pk)).as_tuple()
    proof_wire = p2.as_tuple()
    pub = eth.inputs([33])
    assert verifier.verify(eth.VerifyingKey.from_tuple(vk_wire).to_verifying_key(), pub, eth.Proof.from_tuple(proof_wire).to_proof())
    assert not verifier.verify(eth.VerifyingKey.from_tuple(vk_wire).to_verifying_key(), [34], eth.Proof.from_tuple(proof_wire).to_proof())
    assert eth.VerifyingKey.from_proving_key(pk).as_tuple() == vk_wire


def test_cpp_ethereum_views_match_python(golden):
    """host/ark_circom_ethereum.hpp (C++ mirror of src/ethereum.rs) against circom_compat_b200/ethereum.py on the reference's
    test.zkey and a golden proof: every U256 word of the verifying key, proof, calldata and inputs; the way back
    (VerifyingKey / Proof / Inputs -> ark types, the reference's convert_* tests) and check_proof on the round-tripped objects."""
    import subprocess
    from circom_compat_b200 import Proof, read_zkey
    from circom_compat_b200 import ethereum as eth
    zk = os.path.join(ROOT, 'tests', 'golden', 'test.zkey')
    pk, _ = read_zkey(zk)
    vk = eth.VerifyingKey.from_proving_key(pk)
    for case in golden['test_zkey']['proofs']:
        out = subprocess.check_output([HOST_BIN, '--ethereum', zk, case['proof_hex'], '33'], text=True)
        kv = dict(line.split('=', 1) for line in out.split())
        ep = eth.Proof.from_proof(Proof(bytes.fromhex(case['proof_hex'])))

        def h1(g): return ','.join('%064x' % v for v in g.as_tuple())
        def h2(g): t = g.as_tuple(); return ','.join('%064x' % v for v in (t[0][0], t[0][1], t[1][0], t[1][1]))
        assert kv['vk.alpha1'] == h1(vk.alpha1) and kv['vk.beta2'] == h2(vk.beta2) and kv['vk.gamma2'] == h2(vk.gamma2) and kv['vk.delta2'] == h2(vk.delta2)
        assert [kv['vk.ic[%d]' % i] for i in range(len(vk.ic))] == [h1(p) for p in vk.ic]
        assert kv['proof.a'] == h1(ep.a) and kv['proof.b'] == h2(ep.b) and kv['proof.c'] == h1(ep.c)
        assert kv['calldata'] == ep.calldata().hex()
        assert kv['inputs[0]'] == eth.point_to_u256(33).hex()
        assert kv['roundtrip'] == '1' and kv['verified'] == '1'
    bad = subprocess.check_output([HOST_BIN, '--ethereum', zk, golden['test_zkey']['proofs'][0]['proof_hex'], '34'], text=True)
    assert 'roundtrip=1' in bad and 'verified=0' in bad
    # a coordinate that is not a canonical Fq element cannot come back (u256_to_point's expect in the reference)
    r = subprocess.run([HOST_BIN, '--ethereum', zk, 'ff' * 256, '33'], capture_output=True, text=True)
    assert r.returncode == 1 and 'canonical' in r.stderr


def test_reference_witness_kats_through_the_builder(golden):
    """The four witnesses the reference's witness-calculator tests pin (src/witness/witness_calculator.rs:260-311: multiplier_1/2/3 on
    mycircuit, safe_multipler on circuit2; two of them wrap around the field) fed through the builder mirror: each satisfies its
    .r1cs (read by the product's reader), yields the public inputs circuit.rs:18-26 defines, and the snarkjs witness.wtns fixture
    equals the reference-held JSON element for element - a known answer for read_wtns that does not come from this repository."""
    from circom_compat_b200 import CircomConfig, CircomBuilder, read_wtns
    from circom_compat_b200.zkey import R_MOD
    g = os.path.join(ROOT, 'tests', 'golden')
    k = golden['witness_kats']
    assert k['mycircuit_witness_json'] == k['multiplier'][0] == ['1', '33', '3', '11']
    for wit, inp in zip(k['multiplier'], k['multiplier_inputs']):
        wit = [int(x) for x in wit]
        a, b = int(inp['a']), int(inp['b'])
        assert wit == [1, a * b % R_MOD, a % R_MOD, b]                       # c <== a * b, reduced mod r by the calculator
        builder = CircomBuilder.new(CircomConfig.new(lambda inputs, wit=wit: wit, os.path.join(g, 'mycircuit.r1cs')))
        builder.push_input('a', a); builder.push_input('b', b)
        circom = builder.build()                                            # raises on an unsatisfied constraint
        assert circom.witness == wit and circom.get_public_inputs() == [wit[1]]
    safe = [int(x) for x in k['safe_multiplier']]
    assert len(safe) == 132
    assert read_wtns(open(os.path.join(g, 'circuit2_witness.wtns'), 'rb').read()) == safe
    c2 = CircomBuilder.new(CircomConfig.new(lambda inputs: safe, os.path.join(g, 'circuit2.r1cs'))).build()
    assert c2.get_public_inputs() == [33]
    tampered = list(safe); tampered[5] = (tampered[5] + 1) % R_MOD
    with pytest.raises(ValueError):
        CircomBuilder.new(CircomConfig.new(lambda inputs: tampered, os.path.join(g, 'circuit2.r1cs'))).build()
