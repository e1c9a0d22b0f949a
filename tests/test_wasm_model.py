"""The plain-Python circom 2 witness model (tests/wasm_model.py) pinned to known answers that do not come from this
repository: the reference's witness-calculator KATs (multiplier_1/2/3 and safe_multipler of
src/witness/witness_calculator.rs), the snarkjs witness.wtns of circuit2, the published FNV-1a 64 values, and the
refusal of circom 1 and float modules.  The GPU tests then hold the device interpreter to this model."""
import json
import os

import pytest

import wasm_asm as A
import wasm_model as M
from circom_compat_b200.r1cs import read_wtns

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _wasm(name):
    return open(os.path.join(GOLDEN, name), 'rb').read()


@pytest.fixture(scope='module')
def mycircuit():
    return M.Calculator(_wasm('mycircuit.wasm'))


@pytest.fixture(scope='module')
def circuit2():
    return M.Calculator(_wasm('circuit2.wasm'))


def test_fnv_of_the_input_names():
    assert M.fnv1a64('a') == 0xaf63dc4c8601ec8c and M.fnv1a64('b') == 0xaf63df4c8601f1a5
    assert M.fnv1a64('') == 0xcbf29ce484222325
    from circom_compat_b200.witness import fnv
    assert fnv('a') == (0xaf63dc4c, 0x8601ec8c)


def test_model_reads_the_field_and_sizes(mycircuit, circuit2):
    for c, size in ((mycircuit, 4), (circuit2, 132)):
        assert c.prime == M.R_MOD and c.n32 == 8 and c.version == 2
        assert c.witness_size == size and c.input_size == 2


def test_model_multiplier_kats(golden, mycircuit):
    k = golden['witness_kats']
    for n, (wit, inp) in enumerate(zip(k['multiplier'], k['multiplier_inputs'])):
        fixture = json.load(open(os.path.join(GOLDEN, f'mycircuit-input{n + 1}.json')))
        assert {x: int(v) for x, v in fixture.items()} == {x: int(v) for x, v in inp.items()}
        st, w = mycircuit.calculate([(x, [int(v)]) for x, v in fixture.items()])
        assert st == M.OK and w == [int(x) for x in wit]


def test_model_safe_multiplier_kat_and_wtns(golden, circuit2):
    st, w = circuit2.calculate([('a', [3]), ('b', [11])])
    assert st == M.OK
    assert w == [int(x) for x in golden['witness_kats']['safe_multiplier']]
    assert w == [int(x) for x in json.load(open(os.path.join(GOLDEN, 'safe-circuit-witness.json')))]
    assert w == read_wtns(_wasm('circuit2_witness.wtns'))


def test_model_circuit2_rejects_wide_and_singular_inputs(circuit2):
    # CheckBits(64) fails for a >= 2^64 and (a - 1) * inv === 1 for a = 1: both are circom asserts (code 4)
    for a in (1 << 64, 1, -5):
        st, w = circuit2.calculate([('a', [a]), ('b', [11])])
        assert st == M.EXCEPTION + 4 and w is None


def test_model_reduces_inputs_mod_r(mycircuit):
    st, w = mycircuit.calculate([('a', [M.R_MOD + 3]), ('b', [-11])])
    assert st == M.OK and w == [1, 3 * (M.R_MOD - 11) % M.R_MOD, 3, M.R_MOD - 11]


def test_model_refuses_circom1_and_floats():
    with pytest.raises(M.Refused, match='env.memory'):
        M.Module(_wasm('complex-circuit-10000-10000.wasm'))
    flt = A.module([A.Func([A.F32, A.F32], [A.F32], A.lget(0) + A.lget(1) + b'\x92', export='f')])
    with pytest.raises(M.Refused):
        M.Module(flt, protocol=False)
    fop = A.module([A.Func([A.I32], [A.I32], A.lget(0) + b'\x41\x00' + b'\x6a', export='ok'),
                    A.Func([A.I64], [A.I32], A.lget(0) + b'\xb4' + b'\xa8', export='f')])   # f32.convert_i64_s
    with pytest.raises(M.Refused, match=r'function 1: opcode 0xb4'):
        M.Module(fop, protocol=False).body(1)
    noexp = A.module([A.Func([], [A.I32], b'\x41\x08', export='getFieldNumLen32')], memory=(1, None))
    with pytest.raises(M.Refused, match='does not export the circom 2 function'):
        M.Module(noexp)


def test_model_integer_edges():
    mn = 1 << 31
    f = A.module([A.Func([A.I32, A.I32], [A.I32], A.lget(0) + A.lget(1) + bytes([op]), export=f'op{op:02x}')
                  for op in (0x6d, 0x6f, 0x74)])
    assert M.run_function(f, 'op6d', [mn, M.M32]) == (M.OVERFLOW, None)
    assert M.run_function(f, 'op6d', [5, 0]) == (M.DIV_ZERO, None)
    assert M.run_function(f, 'op6f', [mn, M.M32]) == (M.OK, [0])
    assert M.run_function(f, 'op6d', [(-7) & M.M32, 2]) == (M.OK, [(-3) & M.M32])
    assert M.run_function(f, 'op6f', [(-7) & M.M32, 2]) == (M.OK, [(-1) & M.M32])
    assert M.run_function(f, 'op74', [1, 33]) == (M.OK, [2])
