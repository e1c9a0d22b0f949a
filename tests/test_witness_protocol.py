"""The device witness driver (b2g_witness_calculate: mode 1 of csrc/wasm.cu's wasm_kernel, driver_next, the value
staging, the chunked copy-back and wasm_to_mont_kernel) on hand-built circom 2 modules (tests/circom2_synth.py).

The golden circuits only ever set scalar inputs, two values per lane, into at most 132 wires.  Here the modules have
input arrays of 1 to 20 000 elements under several names, witnesses of 1 to 2^17 + 1 wires, a chunk whose output passes
2^32 bytes, and a fault switch per lane that makes each lane end with its own circom exception, the protocol status or
fuel exhaustion.  Every lane's status and witness row is compared with plain integer arithmetic (sampled lanes where the
whole batch would take the host too long), and sampled lanes with the Python model of tests/wasm_model.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import circom2_synth as S
import wasm_model as M
from circom_compat_b200 import (B2gError, Groth16, R1CS, R1CSFile, WasmModule, WitnessCalculator, WitnessError,
                                fr_from_mont, release)
from circom_compat_b200 import _native as N
from circom_compat_b200.witness import fnv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = M.R_MOD
R_TOP = R >> 224                     # the top word of r: values whose top word is below it are below r


def _mont(xs):
    """canonical ints -> the Montgomery rows b2g_witness_calculate writes (uint64, 4 words per element)"""
    return np.frombuffer(b''.join(((x << 256) % R).to_bytes(32, 'little') for x in xs), dtype=np.uint64)


def _calc(ctx, s, **limits):
    c = WitnessCalculator(s.wasm, ctx)
    if limits:
        c.set_limits(**limits)
    return c


def _lane_bytes(c, n_values, n_wit):
    """the per-lane device bytes run_lanes budgets for (csrc/wasm.cu lane_bytes)"""
    lim = c.limits
    return lim.max_pages * 65536 + lim.stack_slots * 8 + lim.max_depth * 8 + 32 * n_values + 32 * n_wit + 4


def _abi(c, s, vals):
    """b2g_witness_calculate straight from a (count, n_values, 8) uint32 array of canonical values, for batches whose
    Python dicts would take the host longer than the device"""
    count = vals.shape[0]
    hashes = np.array([(lambda m, l: (m << 32) | l)(*fnv(n)) for n, _ in s.signals], dtype=np.uint64)
    counts = np.array([size for _, size in s.signals], dtype=np.uint32)
    vals = np.ascontiguousarray(vals, dtype=np.uint32)
    w = np.zeros((count, 4 * s.n_wit), dtype=np.uint64)
    st = np.zeros(count, dtype=np.uint32)
    p = lambda a: C.c_void_p(a.ctypes.data) if a.size else None   # noqa: E731
    N.check(N.lib().b2g_witness_calculate(c.ctx._h, c._h, count, len(s.signals), p(hashes), p(counts), p(vals), 0,
                                          p(w), p(st)))
    return w, st


def _random_values(rng, count, n_values):
    """(count, n_values, 8) uint32 canonical values below r, edge values included"""
    v = rng.integers(0, 1 << 32, size=(count, n_values, 8), dtype=np.uint64).astype(np.uint32)
    v[..., 7] %= R_TOP
    if v.size:
        flat = v.reshape(-1, 8)
        flat[::7] = 0
        flat[3::11] = np.frombuffer((R - 1).to_bytes(32, 'little'), dtype=np.uint32)
    return v


def _ints(row):
    """a (n_values, 8) uint32 row -> ints"""
    return [int.from_bytes(x.tobytes(), 'little') for x in row]


def _split(s, ints):
    out, k = {}, 0
    for n, size in s.signals:
        out[n] = ints[k:k + size]
        k += size
    return out


def _check_rows(s, w, st, inputs_of, lanes):
    for i in lanes:
        ins = inputs_of(i)
        assert st[i] == s.expected_status(ins), (i, int(st[i]))
        if st[i] == M.OK:
            assert np.array_equal(w[i], _mont(s.expected(ins))), i
        else:
            assert not w[i].any(), i


def _model_rows(s, w, st, inputs_of, lanes, **limits):
    model = M.Calculator(s.wasm, **limits)
    for i in lanes:
        ins = inputs_of(i)
        ms, mw = model.calculate([(n, list(v) if isinstance(v, (list, tuple)) else [v]) for n, v in ins.items()])
        assert st[i] == ms, (i, int(st[i]), ms)
        if ms == M.OK:
            assert fr_from_mont(w[i]) == mw, i


def _sample(count, rng, k=16):
    edges = {0, 1, 30, 31, 32, 33, count // 2, count - 33, count - 32, count - 2, count - 1}
    return sorted({i for i in edges if 0 <= i < count} | set(rng.sample(range(count), min(k, count))))


# ------------------------------------------------------------------------------------------------ arrays and names
ARRAYS = [('in', 1), ('pair', 2), ('tri', 3), ('w31', 31), ('w32', 32), ('w33', 33), ('big', 1000)]


def test_arrays_under_many_names_in_any_order(ctx):
    s = S.Synth(ARRAYS, n_wit=1 + 1102 + 300)
    c = _calc(ctx, s)
    assert (c.witness_size, c.input_size) == (s.n_wit, 1102)
    rng = random.Random(17)
    edge = [0, 1, R - 1, R, R + 1, -1, -R - 5, (1 << 256) - 1]
    lanes = [{n: [rng.choice(edge) if rng.random() < 0.2 else rng.randrange(R) for _ in range(size)] for n, size in ARRAYS}
             for _ in range(33)]
    # numpy integers and decimal strings inside arrays are accepted as the integers they spell
    lanes[5]['tri'] = [np.uint64(7), np.int64(-3), str(R + 2)]
    lanes[6]['pair'] = ['12345678901234567890123456789', '-4']
    plain = [{n: [int(x) for x in v] for n, v in ins.items()} for ins in lanes]
    rows = []
    for seed in (1, 2, 3):
        order = [n for n, _ in ARRAYS]
        random.Random(seed).shuffle(order)
        w, st = c.calculate_witnesses([{n: ins[n] for n in order} for ins in lanes])
        rows.append(w)
        _check_rows(s, w, st, lambda i: plain[i], range(33))
    assert all(np.array_equal(rows[0], r) for r in rows[1:])
    for i in (0, 5, 6, 32):
        want = s.expected(plain[i])
        order = [n for n, _ in ARRAYS][::-1]
        assert c.calculate_witness({n: lanes[i][n] for n in order}) == want
        assert c.calculate_witness_element(list(lanes[i].items())) == want
    _model_rows(s, rows[0], np.zeros(33, dtype=np.uint32), lambda i: plain[i], [0, 32])
    c.close()


# ------------------------------------------------------------------------------------------------ value counts
_MODULES = {}


def _counts_module(n_values):
    if n_values not in _MODULES:
        sig = [] if n_values == 0 else [('a', n_values)] if n_values == 1 else [('a', n_values // 2), ('b', n_values - n_values // 2)]
        _MODULES[n_values] = S.Synth(sig, n_wit=1 + n_values + 40)
    return _MODULES[n_values]


@pytest.mark.parametrize('count', [1, 31, 32, 33, 1024])
@pytest.mark.parametrize('n_values', [0, 1, 2, 3, 1000, 20000])
def test_value_counts_at_lane_counts(ctx, n_values, count):
    s = _counts_module(n_values)
    c = _calc(ctx, s)
    rng = np.random.default_rng(n_values * 1031 + count)
    vals = _random_values(rng, count, n_values)
    w, st = _abi(c, s, vals)
    assert not st.any()
    inputs_of = lambda i: _split(s, _ints(vals[i]))     # noqa: E731
    full = count * (n_values + s.n_wit) <= 2_500_000
    lanes = range(count) if full else _sample(count, random.Random(count))
    _check_rows(s, w, st, inputs_of, lanes)
    if n_values <= 1000:
        _model_rows(s, w, st, inputs_of, sorted({0, count - 1}))
    if n_values and count > 1:       # the Python entry point stages the same values the same way
        wp, stp = c.calculate_witnesses([{n: v for n, v in inputs_of(i).items()} for i in (0, count - 1)])
        assert not stp.any() and np.array_equal(wp, w[[0, count - 1]])
    c.close()


# ------------------------------------------------------------------------------------------------ witness sizes
@pytest.mark.parametrize('n_wit,signals', [(1, []), (2, []), (132, [('a', 2), ('b', 3)]), (4097, [('a', 5)]),
                                           ((1 << 17) + 1, [('a', 3), ('b', 1)])])
def test_witness_sizes(ctx, n_wit, signals):
    s = S.Synth(signals, n_wit=n_wit)
    c = _calc(ctx, s)
    assert c.witness_size == n_wit
    count = 33
    rng = random.Random(n_wit)
    lanes = [{n: [rng.randrange(R) for _ in range(size)] for n, size in signals} for _ in range(count)]
    w, st = c.calculate_witnesses(lanes)
    assert w.shape == (count, 4 * n_wit) and not st.any()
    _check_rows(s, w, st, lambda i: lanes[i], range(count) if n_wit <= 4097 else [0, 1, 31, 32])
    if n_wit <= 132:
        _model_rows(s, w, st, lambda i: lanes[i], [0, 32])
    c.close()


def test_one_chunk_of_more_than_4_gib_of_witness(ctx):
    """2^15 lanes x 4097 wires x 32 B = 2^32 + 2^20 bytes written by one chunk: the copy-back offsets and
    wasm_to_mont_kernel's element index must not wrap at 32 bits"""
    s = S.Synth([('x', 1)], n_wit=4097)
    count = 1 << 15
    c = _calc(ctx, s, max_pages=s.pages)
    c.set_limits(budget_bytes=_lane_bytes(c, 1, s.n_wit) * count)          # exactly one chunk
    assert count * s.n_wit * 32 > 1 << 32
    rng = random.Random(15)
    xs = [rng.randrange(R) for _ in range(count)]
    w, st = c.calculate_witnesses([{'x': x} for x in xs])
    assert not st.any()
    # every lane: wire 0, its input and its last wire.  Each wire is alpha + beta x, so the last one is cheap per lane.
    coef = [(1, 0), (0, 1)]
    for k in range(2, s.n_wit):
        a, b = coef[k - 1], coef[S.pattern(k)]
        coef.append(((a[0] + b[0]) % R, (a[1] + b[1]) % R))
    alpha, beta = coef[-1]
    assert np.array_equal(w[:, :4], np.tile(_mont([1]), (count, 1)))
    assert np.array_equal(w[:, 4:8], _mont(xs).reshape(count, 4))
    assert np.array_equal(w[:, -4:], _mont([(alpha + beta * x) % R for x in xs]).reshape(count, 4))
    _check_rows(s, w, st, lambda i: {'x': xs[i]}, _sample(count, rng, 8))
    c.close()


# ------------------------------------------------------------------------------------------------ chunks and statuses
FAULT_SIGNALS = [('mode', 1), ('x', 3), ('y', 2)]
FUEL = 200_000


def _fault_lanes(count, faults, seed):
    rng = random.Random(seed)
    return [{'mode': faults.get(i, 0), 'x': [rng.randrange(R) for _ in range(3)], 'y': [rng.randrange(R), R - 1]}
            for i in range(count)]


def test_chunks_of_one_and_two_warps_and_a_partial_last_chunk(ctx):
    s = S.Synth(FAULT_SIGNALS, n_wit=90, mode='mode')
    faults = {0: 4, 31: 3, 32: 1, 63: 8, 64: 6, 99: 2}
    lanes = _fault_lanes(100, faults, 8)
    whole_c = _calc(ctx, s, fuel=FUEL)
    whole, st0 = whole_c.calculate_witnesses(lanes)
    _check_rows(s, whole, st0, lambda i: lanes[i], range(100))
    per = _lane_bytes(whole_c, 6, s.n_wit)
    for lanes_per_chunk in (32, 64):                    # 32, 32, 32, 4 and 64, 36
        c = _calc(ctx, s, fuel=FUEL, budget_bytes=per * lanes_per_chunk + per - 1)
        w, st = c.calculate_witnesses(lanes)
        assert w.tobytes() == whole.tobytes() and np.array_equal(st, st0)
        c.close()
    whole_c.close()


def test_each_lane_gets_its_own_status(ctx):
    """one call in chunks of 32 lanes: circom's exception codes 1, 2, 3, 4 and 6, the protocol status and fuel
    exhaustion at the first and last lanes and on both sides of each chunk boundary"""
    s = S.Synth(FAULT_SIGNALS, n_wit=64, mode='mode')
    count = 130
    faults = {0: 1, 31: 2, 32: 3, 63: 4, 64: 6, 95: 8, 96: 9, 127: 9, 128: 8, 129: 6, 50: 4, 51: 1, 52: 2}
    lanes = _fault_lanes(count, faults, 9)
    c = _calc(ctx, s, fuel=FUEL)
    c.set_limits(budget_bytes=_lane_bytes(c, 6, s.n_wit) * 32)
    w, st = c.calculate_witnesses(lanes)
    assert [int(x) for x in st] == [S.MODES[faults.get(i, 0)] for i in range(count)]
    _check_rows(s, w, st, lambda i: lanes[i], range(count))
    _model_rows(s, w, st, lambda i: lanes[i], [0, 1, 31, 32, 33, 63, 64, 95, 96, 128], fuel=FUEL)
    names = {1: 'Signal not found', 2: 'Too many signals set', 3: 'Signal already set', 4: 'Assert Failed',
             6: 'Input signal array access exceeds the size', 8: "getWitnessSize disagrees", 9: 'fuel'}
    for mode, text in names.items():
        with pytest.raises(WitnessError, match=text) as e:
            c.calculate_witness(_fault_lanes(1, {0: mode}, mode)[0])
        assert e.value.status == S.MODES[mode]
    ok = _fault_lanes(1, {}, 3)[0]
    assert c.calculate_witness(ok) == s.expected(ok)
    c.close()


def test_module_wide_faults(ctx):
    """getWitnessSize reporting N + 1 after init ends every lane with the protocol status; a getInputSize below the
    values passed ends every lane with code 2"""
    lanes = [{'a': [1, 2], 'b': [3]}] * 33
    for s, status in ((S.Synth([('a', 2), ('b', 1)], n_wit=20, protocol_fault=True), M.PROTOCOL),
                      (S.Synth([('a', 2), ('b', 1)], n_wit=20, input_size=2), M.EXCEPTION + 2)):
        c = _calc(ctx, s)
        assert c.witness_size == 20
        w, st = c.calculate_witnesses(lanes)
        assert (st == status).all() and not w.any()
        assert M.Calculator(s.wasm).calculate(list(lanes[0].items()))[0] == status
        c.close()


# ------------------------------------------------------------------------------------------------ refusals
def _last_error():
    return N.lib().b2g_last_error().decode()


def test_abi_and_host_refusals_leave_the_calculator_working(ctx):
    s = S.Synth([('a', 2), ('b', 1)], n_wit=30)
    c = _calc(ctx, s)
    L = N.lib()
    good = [{'a': [5, 6], 'b': [7]}, {'a': [R - 1, 0], 'b': [1]}]
    want = np.stack([_mont(s.expected(x)) for x in good])

    def still_works():
        w, st = c.calculate_witnesses(good)
        assert not st.any() and np.array_equal(w, want)
    still_works()
    hashes = np.array([(lambda m, l: (m << 32) | l)(*fnv(n)) for n, _ in s.signals], dtype=np.uint64)
    counts = np.array([2, 1], dtype=np.uint32)
    out = np.zeros((2, 4 * s.n_wit), dtype=np.uint64)
    st = np.zeros(2, dtype=np.uint32)
    p = lambda a: C.c_void_p(a.ctypes.data)   # noqa: E731
    # a value at or above r at a non-zero index, named by its index
    for bad in (R, R + 1, (1 << 256) - 1):
        for e in (1, 4, 5):
            vals = np.zeros((6, 8), dtype=np.uint32)
            vals[e] = np.frombuffer(bad.to_bytes(32, 'little'), dtype=np.uint32)
            rc = L.b2g_witness_calculate(ctx._h, c._h, 2, 2, p(hashes), p(counts), p(vals), 0, p(out), p(st))
            assert rc == N.B2G_E_INPUT and _last_error() == f"values_canon[{e}] is not below r", (bad, e)
            still_works()
    vals = np.zeros((6, 8), dtype=np.uint32)
    # more than 2^24 values per witness: refused before the values are read
    big = np.array([1 << 24, 1], dtype=np.uint32)
    for cnt in (np.array([(1 << 24) + 1], dtype=np.uint32), big):
        rc = L.b2g_witness_calculate(ctx._h, c._h, 1, len(cnt), p(hashes), p(cnt), p(vals), 0, p(out), p(st))
        assert rc == N.B2G_E_SHAPE and _last_error() == "too many input values"
        still_works()
    # null pointers
    args = [ctx._h, c._h, 2, 2, p(hashes), p(counts), p(vals), 0, p(out), p(st)]
    for k in (0, 1, 4, 5, 6, 8, 9):
        a = list(args)
        a[k] = None
        rc = L.b2g_witness_calculate(*a)
        assert rc == N.B2G_E_SHAPE and _last_error() == "null pointer", k
        still_works()
    # a module loaded as a plain module
    plain = WasmModule(s.wasm, ctx)
    rc = L.b2g_witness_calculate(ctx._h, plain._h, 2, 2, p(hashes), p(counts), p(vals), 0, p(out), p(st))
    assert rc == N.B2G_E_SHAPE and 'not loaded as a circom 2 witness calculator' in _last_error()
    plain.close()
    # a module that claims about 5 x 10^8 wires: too many protocol calls per witness, refused before any allocation
    huge = S.Synth([('a', 1)], n_wit=2, claimed_size=500_000_000)
    hc = _calc(ctx, huge)
    assert hc.witness_size == 500_000_000
    h1 = np.array([hashes[0]], dtype=np.uint64)
    one = np.array([1], dtype=np.uint32)
    rc = L.b2g_witness_calculate(ctx._h, hc._h, 1, 1, p(h1), p(one), p(vals), 0, p(out), p(st))
    assert rc == N.B2G_E_SHAPE and _last_error() == "too many calls per witness"
    hc.close()
    still_works()
    # the Python side: inputs of different names, lengths or order are refused before anything runs
    for other in ({'a': [1, 2], 'b': [3, 4]}, {'a': [1], 'b': [3]}, {'b': [3], 'a': [1, 2]}, {'a': [1, 2], 'c': [3]}):
        with pytest.raises(ValueError, match='does not have the names and lengths'):
            c.calculate_witnesses([good[0], other])
        still_works()
    # negative values, values >= r and numpy integers are reduced mod r
    w, st = c.calculate_witnesses([{'a': [5 - R, R + 6], 'b': [np.int64(7)]}, {'a': [-1, 2 * R], 'b': np.uint64(1)}])
    assert not st.any() and np.array_equal(w, want)
    c.close()


# ------------------------------------------------------------------------------------------------ end to end
E2E = [('pub', 2), ('x', 3), ('y', 33)]


def _e2e_lanes(count, seed):
    rng = random.Random(seed)
    return [{'pub': [rng.randrange(1 << 64) for _ in range(2)], 'x': [rng.randrange(R) for _ in range(3)],
             'y': [rng.randrange(1 << 64) for _ in range(33)]} for _ in range(count)]


def test_array_witnesses_prove_and_verify(ctx):
    s = S.Synth(E2E, n_wit=200)
    c = _calc(ctx, s)
    lanes = _e2e_lanes(64, 4)
    wm, st = c.calculate_witnesses(lanes)
    _check_rows(s, wm, st, lambda i: lanes[i], range(64))
    circuit = R1CS.from_file(R1CSFile.new(s.r1cs(n_public=2))).to_circuit()
    rng = random.Random(99)
    pk = Groth16.generate_random_parameters_with_reduction(circuit, rng, ctx)
    cm = circuit.matrices()
    proofs = Groth16.create_proofs(pk, [(rng.randrange(1, R), rng.randrange(1, R)) for _ in lanes], cm, wm, ctx)
    pubs = [ins['pub'] for ins in lanes]
    assert Groth16.verify_many(pk, pubs, proofs, ctx) == [True] * 64
    pubs[7] = [pubs[7][0], pubs[7][1] + 1]
    assert Groth16.verify_many(pk, pubs, proofs, ctx) == [k != 7 for k in range(64)]
    release(pk)
    release(cm)
    c.close()


def test_cpp_mirror_with_array_inputs_equals_python(ctx, tmp_path):
    """B2G_WITNESS=<module> groth16_bench <r1cs> pub=.. pub=.. x=.. (repeated names fill the arrays) count: the C++
    WitnessCalculator's witnesses prove and verify there, and equal the Python ones word for word"""
    s = S.Synth(E2E, n_wit=200)
    (tmp_path / 'c.wasm').write_bytes(s.wasm)
    (tmp_path / 'c.r1cs').write_bytes(s.r1cs(n_public=2))
    ins = _e2e_lanes(1, 5)[0]
    ins['x'][1] = -12345                       # a leading - maps to r - |v|
    out = tmp_path / 'w.bin'
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    env = dict(os.environ, B2G_WITNESS=str(tmp_path / 'c.wasm'), B2G_WITNESS_OUT=str(out))
    args = [f'{n}={v}' for n in ('y', 'pub', 'x') for v in ins[n]]      # not in table order
    p = subprocess.run([exe, str(tmp_path / 'c.r1cs')] + args + ['12'], env=env, capture_output=True, text=True,
                       timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert 'verified 12/12' in p.stdout, p.stdout
    got = np.fromfile(out, dtype=np.uint64).reshape(12, -1)
    c = _calc(ctx, s)
    want, st = c.calculate_witnesses([ins] * 12)
    assert not st.any() and np.array_equal(got, want)
    assert np.array_equal(want[0], _mont(s.expected(ins)))
    c.close()
