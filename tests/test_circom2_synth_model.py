"""The hand-built circom 2 modules of tests/circom2_synth.py on the Python model (no GPU): the model's witness and lane
status must equal the plain integer formula for every signal shape, input order and fault switch, so the device tests
of tests/test_witness_protocol.py have two yardsticks that do not depend on the device."""
import random

import pytest

import circom2_synth as S
import wasm_model as M
from circom_compat_b200 import R1CS, R1CSFile

R = M.R_MOD


def _run(s, inputs, **limits):
    return M.Calculator(s.wasm, **limits).calculate([(n, v if isinstance(v, list) else [v]) for n, v in inputs])


def _values(rng, size):
    edge = [0, 1, R - 1, R, R + 1, -1, -R, (1 << 256) - 1, 1 << 255]
    return [rng.choice(edge) if rng.random() < 0.3 else rng.randrange(-R, 2 * R) for _ in range(size)]


@pytest.mark.parametrize('sizes', [[1], [2], [3], [31, 32, 33], [1, 2, 3, 33]])
def test_model_equals_the_formula_for_arrays_in_any_order(sizes):
    signals = [(f's{k}_{n}', n) for k, n in enumerate(sizes)]
    s = S.Synth(signals, n_wit=1 + sum(sizes) + 70)
    c = M.Calculator(s.wasm)
    assert (c.version, c.n32, c.prime, c.witness_size, c.input_size) == (2, 8, R, s.n_wit, sum(sizes))
    rng = random.Random(sum(sizes))
    for _ in range(2):
        ins = {n: _values(rng, size) for n, size in signals}
        order = list(ins)
        rng.shuffle(order)
        st, w = c.calculate([(n, ins[n]) for n in order])
        assert st == M.OK and w == s.expected(ins)
        assert all(0 <= x < R for x in w) and w[0] == 1


def test_model_equals_the_formula_without_inputs_and_at_the_smallest_sizes():
    for n_wit in (1, 2, 3, 40):
        s = S.Synth([], n_wit=n_wit)
        assert _run(s, []) == (M.OK, s.expected({}))
    s = S.Synth([('x', 1)])
    assert _run(s, [('x', 7)]) == (M.OK, [1, 7])


def test_every_fault_mode_gives_its_status_on_the_model():
    s = S.Synth([('mode', 1), ('x', 3), ('y', 2)], n_wit=60, mode='mode')
    for m in sorted(S.MODES) + [5, 7, 10]:
        ins = {'mode': m, 'x': [3, 4, 5], 'y': [R - 1, 9]}
        st, w = _run(s, list(ins.items()), fuel=200000)
        assert st == s.expected_status(ins) == S.MODES.get(m, M.OK), m
        assert w == (s.expected(ins) if st == M.OK else None)


def test_the_module_switches_and_the_protocol_check():
    ins = [('a', [1, 2]), ('b', [3])]
    # more values than getInputSize: code 2 once the first input_size are in
    s = S.Synth([('a', 2), ('b', 1)], n_wit=9, input_size=2)
    assert _run(s, ins) == (M.EXCEPTION + 2, None) and s.expected_status(dict(ins)) == M.EXCEPTION + 2
    # getWitnessSize reports N + 1 once init has run: the model refuses it as the device does
    s = S.Synth([('a', 2), ('b', 1)], n_wit=9, protocol_fault=True)
    c = M.Calculator(s.wasm)
    assert c.witness_size == 9 and c.calculate(ins) == (M.PROTOCOL, None)
    # an unknown name, an index past the size, an element set twice
    s = S.Synth([('a', 2), ('b', 1)], n_wit=9)
    c = M.Calculator(s.wasm)
    assert c.calculate([('a', [1, 2]), ('c', [3])])[0] == M.EXCEPTION + 1
    assert c.calculate([('a', [1, 2, 3])])[0] == M.EXCEPTION + 6
    assert c.calculate([('a', [1, 2]), ('a', [3])])[0] == M.EXCEPTION + 3
    assert c.calculate([('b', [3]), ('a', [1, 2])]) == (M.OK, s.expected(dict(ins)))
    # the size reported outright: probed and returned the same, so no protocol error
    s = S.Synth([('a', 1)], n_wit=2, claimed_size=500_000_000)
    assert M.Calculator(s.wasm).witness_size == 500_000_000


def test_r1cs_of_the_synthetic_circuit_reads_back_and_holds():
    s = S.Synth([('pub', 2), ('x', 3), ('y', 33)], n_wit=160)
    r1cs = R1CS.from_file(R1CSFile.new(s.r1cs(n_public=2)))
    assert (r1cs.num_inputs, r1cs.num_variables, len(r1cs.constraints)) == (3, 160, 160 - 1 - 38)
    rng = random.Random(3)
    w = s.expected({'pub': [5, 6], 'x': _values(rng, 3), 'y': _values(rng, 33)})

    def holds(w):
        return all(sum(c * w[i] for i, c in a) * sum(c * w[i] for i, c in b) % R == sum(c * w[i] for i, c in cc) % R
                   for a, b, cc in r1cs.constraints)
    assert holds(w)
    w[100] = (w[100] + 1) % R
    assert not holds(w)
    assert all(S.pattern(k) < k for k in range(1, 1 << 18))
