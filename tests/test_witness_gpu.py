"""circom 2 witnesses on the GPU (csrc/wasm.cu): every opcode of the integer subset at its edge values, every per-lane
limit, the reference's fixtures at many counts and chunkings, and the whole flow from the .wasm to verified proofs.
The yardstick is the plain-Python model of tests/wasm_model.py, which shares nothing with the library's translator."""
import os
import random
import subprocess

import numpy as np
import pytest

import wasm_asm as A
import wasm_model as M
from circom_compat_b200 import (CircomBuilder, CircomConfig, Groth16, R1CS, R1CSFile, WasmModule, WitnessCalculator,
                                WitnessError, B2gError, fr_from_mont, fr_to_mont, read_wtns, release)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
R = M.R_MOD
M32, M64 = M.M32, M.M64


def _wasm(name):
    return open(os.path.join(GOLDEN, name), 'rb').read()


def _lanes_equal_model(data, name, rows, dev, **limits):
    res, st = dev.run(name, rows)
    for k, row in enumerate(rows):
        ms, mr = M.run_function(data, name, list(row), **limits)
        assert st[k] == ms, (name, row, int(st[k]), ms)
        if ms == M.OK:
            want = mr[0] if mr else 0
            assert int(res[k]) == want, (name, row, hex(int(res[k])), hex(want))


# ------------------------------------------------------------------------------------------------ opcode edges
E32 = [0, 1, M32, 1 << 31, (1 << 31) - 1, 2, 31, 32, 33, 0x12345678, 0xfffffffe]
E64 = [0, 1, M64, 1 << 63, (1 << 63) - 1, 2, 63, 64, 65, 0x123456789abcdef0, M32, 1 << 32]


def _op_module():
    fs = []
    for op in list(range(0x46, 0x50)) + list(range(0x6a, 0x79)):
        fs.append(A.Func([A.I32, A.I32], [A.I32], A.lget(0) + A.lget(1) + bytes([op]), export=f'b{op:02x}'))
    for op in list(range(0x51, 0x5b)):
        fs.append(A.Func([A.I64, A.I64], [A.I32], A.lget(0) + A.lget(1) + bytes([op]), export=f'b{op:02x}'))
    for op in list(range(0x7c, 0x8b)):
        fs.append(A.Func([A.I64, A.I64], [A.I64], A.lget(0) + A.lget(1) + bytes([op]), export=f'b{op:02x}'))
    for op, pt, rt in [(0x45, A.I32, A.I32), (0x67, A.I32, A.I32), (0x68, A.I32, A.I32), (0x69, A.I32, A.I32),
                       (0xc0, A.I32, A.I32), (0xc1, A.I32, A.I32), (0x50, A.I64, A.I32), (0x79, A.I64, A.I64),
                       (0x7a, A.I64, A.I64), (0x7b, A.I64, A.I64), (0xc2, A.I64, A.I64), (0xc3, A.I64, A.I64),
                       (0xc4, A.I64, A.I64), (0xa7, A.I64, A.I32), (0xac, A.I32, A.I64), (0xad, A.I32, A.I64)]:
        fs.append(A.Func([pt], [rt], A.lget(0) + bytes([op]), export=f'u{op:02x}'))
    # select, drop, locals, globals, const
    fs.append(A.Func([A.I32, A.I32, A.I32], [A.I32], A.lget(0) + A.lget(1) + A.lget(2) + b'\x1b', export='select'))
    fs.append(A.Func([A.I64, A.I64, A.I32], [A.I64], A.lget(0) + A.lget(1) + A.lget(2) + b'\x1b', export='select64'))
    fs.append(A.Func([A.I64], [A.I64], A.lget(0) + b'\x24\x00' + A.i64c(7) + b'\x1a' + b'\x23\x00' + A.lget(0) + b'\x7c',
                     export='global'))
    fs.append(A.Func([A.I32], [A.I64], A.i64c(-2) + b'\x21\x01' + A.lget(0) + b'\x22\x02' + b'\x1a' + A.lget(1) + A.lget(2)
                     + b'\xad\x7e', locals_=[A.I64, A.I32], export='locals'))
    return A.module(fs, globals_=[(A.I64, 1, A.i64c(5))])


def test_every_integer_opcode_at_its_edges(ctx):
    data = _op_module()
    dev = WasmModule(data, ctx)
    for name in [e for e in _exports(data)]:
        if name.startswith('b'):
            op = int(name[1:], 16)
            wide = (0x51 <= op <= 0x5a) or op >= 0x7c
            E = E64 if wide else E32
            rows = [(a, b) for a in E for b in E]
        elif name.startswith('u'):
            op = int(name[1:], 16)
            rows = [(a,) for a in (E64 if op in (0x50, 0x79, 0x7a, 0x7b, 0xc2, 0xc3, 0xc4, 0xa7) else E32)]
            rows += [(0x80,), (0x7f,), (0x8000,), (0xff80,)]
        elif name == 'select':
            rows = [(a, b, c) for a in (0, M32) for b in (1, 1 << 31) for c in (0, 1, 2, M32)]
        elif name == 'select64':
            rows = [(a, b, c) for a in (0, M64) for b in (1, 1 << 63) for c in (0, 1, 1 << 31)]
        elif name == 'global':
            rows = [(v,) for v in E64]
        else:
            rows = [(v,) for v in E32]
        _lanes_equal_model(data, name, rows, dev)
    dev.close()


def _exports(data):
    return list(M.Module(data, protocol=False).exports)


def _mem_module():
    pattern = bytes((37 * k + 11) & 0xff for k in range(64))
    fs = []
    for op in (0x28, 0x29, 0x2c, 0x2d, 0x2e, 0x2f, 0x30, 0x31, 0x32, 0x33, 0x34, 0x35):
        rt = A.I32 if op in (0x28, 0x2c, 0x2d, 0x2e, 0x2f) else A.I64
        fs.append(A.Func([A.I32], [rt], A.lget(0) + A.memarg(op), export=f'ld{op:02x}'))
        fs.append(A.Func([A.I32], [rt], A.lget(0) + A.memarg(op, offset=5), export=f'ldo{op:02x}'))
    for op in (0x36, 0x37, 0x3a, 0x3b, 0x3c, 0x3d, 0x3e):
        vt = A.I32 if op in (0x36, 0x3a, 0x3b) else A.I64
        # store, then read back the 12 bytes around the address as one i64: load(a&~3) ^ rotl(load(a&~3 + 4), 17)
        back = (A.lget(0) + A.i32c(-4) + b'\x71' + A.memarg(0x29) + A.lget(0) + A.i32c(-4) + b'\x71' + A.memarg(0x29, 4)
                + A.i64c(17) + b'\x89' + b'\x85')
        fs.append(A.Func([A.I32, vt], [A.I64], A.lget(0) + A.lget(1) + A.memarg(op) + back, export=f'st{op:02x}'))
    fs.append(A.Func([], [A.I32], b'\x3f\x00', export='size'))
    return A.module(fs, memory=(1, 4), data=[(0, pattern), (65536 - 64, pattern)])


def test_loads_and_stores_at_every_alignment_and_the_memory_edge(ctx):
    data = _mem_module()
    dev = WasmModule(data, ctx)
    addrs = list(range(0, 13)) + [65536 - k for k in range(1, 14)] + [65536, M32, M32 - 4]
    for name in _exports(data):
        if name.startswith('ld'):
            _lanes_equal_model(data, name, [(a,) for a in addrs], dev)
        elif name.startswith('st'):
            vals = [0x0123456789abcdef, M64, 0x80, 0x8000]
            op = int(name[2:], 16)
            if op in (0x36, 0x3a, 0x3b):
                vals = [v & M32 for v in vals]
            _lanes_equal_model(data, name, [(a, v) for a in addrs for v in vals], dev)
    _lanes_equal_model(data, 'size', [()] * 3, dev)
    dev.close()


def _control_module():
    # 0: recurse(n) = n == 0 ? 0 : recurse(n - 1) + 1          1: spin(n): loop forever unless n == 0
    # 2: trap(n): unreachable if n != 0                          3: grow(n) = memory.grow(n) + the last word of the memory
    # 4: table(i) = call_indirect type (i32)->i32 of element i  5: ret7(x) = x + 7 (table element 0)   6: none()  (element 1)
    # 7: br_table(i): block nest, the index picks 10, 20, 30 or the default 40
    # 8: ifelse(n): if n then n*2 else n+100 with a result      9: loopsum(n) = 0 + 1 + ... + (n-1) with br_if
    rec = A.lget(0) + b'\x45\x04\x7f' + A.i32c(0) + b'\x05' + A.lget(0) + A.i32c(1) + b'\x6b\x10\x00' + A.i32c(1) + b'\x6a\x0b'
    spin = A.lget(0) + b'\x04\x40\x03\x40\x0c\x00\x0b\x0b' + A.i32c(0)
    trap = A.lget(0) + b'\x04\x40\x00\x0b' + A.i32c(1)
    grow = A.lget(0) + b'\x40\x00\x22\x01' + A.i32c(-1) + b'\x46\x04\x7f' + A.i32c(-1) + b'\x05' + b'\x3f\x00' + \
        A.i32c(16) + b'\x74' + A.i32c(4) + b'\x6b' + A.memarg(0x28) + A.lget(1) + b'\x6a\x0b'
    table = A.i32c(5) + A.lget(0) + b'\x11\x00\x00'
    brt = (b'\x02\x40\x02\x40\x02\x40\x02\x40' + A.lget(0) + b'\x0e\x03\x00\x01\x02\x03\x0b' + A.i32c(10) + b'\x0f\x0b' +
           A.i32c(20) + b'\x0f\x0b' + A.i32c(30) + b'\x0f\x0b' + A.i32c(40))
    ifelse = A.lget(0) + b'\x04\x7f' + A.lget(0) + A.i32c(2) + b'\x6c\x05' + A.lget(0) + A.i32c(100) + b'\x6a\x0b'
    loopsum = (b'\x02\x40\x03\x40' + A.lget(1) + A.lget(0) + b'\x4f\x0d\x01' + A.lget(2) + A.lget(1) + b'\x6a\x21\x02' +
               A.lget(1) + A.i32c(1) + b'\x6a\x21\x01\x0c\x00\x0b\x0b' + A.lget(2))
    fs = [A.Func([A.I32], [A.I32], rec, export='recurse'), A.Func([A.I32], [A.I32], spin, export='spin'),
          A.Func([A.I32], [A.I32], trap, export='trap'), A.Func([A.I32], [A.I32], grow, locals_=[A.I32], export='grow'),
          A.Func([A.I32], [A.I32], table, export='table'), A.Func([A.I32], [A.I32], A.lget(0) + A.i32c(7) + b'\x6a', export='ret7'),
          A.Func([], [], b'', export='none'), A.Func([A.I32], [A.I32], brt, export='br_table'),
          A.Func([A.I32], [A.I32], ifelse, export='ifelse'), A.Func([A.I32], [A.I32], loopsum, locals_=[A.I32, A.I32], export='loopsum')]
    return A.module(fs, memory=(1, None), table=3, elems=[(0, [5, 6])])


def test_control_flow_matches_the_model(ctx):
    data = _control_module()
    dev = WasmModule(data, ctx)
    _lanes_equal_model(data, 'br_table', [(i,) for i in (0, 1, 2, 3, 4, 1000, M32)], dev)
    _lanes_equal_model(data, 'ifelse', [(i,) for i in (0, 1, 5, M32)], dev)
    _lanes_equal_model(data, 'loopsum', [(i,) for i in (0, 1, 2, 100, 1000)], dev)
    _lanes_equal_model(data, 'recurse', [(i,) for i in (0, 1, 10, 200)], dev)
    dev.close()


def test_each_limit_ends_its_own_lane(ctx):
    """a load past memory, runaway recursion, memory.grow past the cap, an endless loop under a small fuel budget,
    unreachable and a bad call_indirect: each lane ends with its own status, its neighbours finish, the call returns"""
    data = _control_module()
    dev = WasmModule(data, ctx)
    dev.set_limits(max_pages=3, max_depth=64, fuel=100000)
    lim = dict(max_pages=3, max_depth=64, fuel=100000)
    rows = [(n,) for n in (0, 10, 62, 63, 64, 1000, 10 ** 9)] * 5
    res, st = dev.run('recurse', rows)
    for (n,), r, s in zip(rows, res, st):     # recurse(n) needs n + 1 frames
        assert (s, r) == ((M.OK, n) if n + 1 <= 64 else (M.STACK, 0)), (n, s, r)
    _lanes_equal_model(data, 'recurse', rows[:7], dev, **lim)
    rows = [(0,), (1,)] * 20
    res, st = dev.run('spin', rows)
    assert list(st) == [M.OK, M.FUEL] * 20
    _lanes_equal_model(data, 'spin', rows[:2], dev, **lim)
    res, st = dev.run('trap', [(0,), (1,), (0,), (7,)])
    assert list(st) == [M.OK, M.UNREACHABLE, M.OK, M.UNREACHABLE] and res[0] == res[2] == 1
    rows = [(0,), (1,), (2,), (3,), (M32,), (1,)]
    res, st = dev.run('grow', rows)          # grow within the cap reads 0 from the new page; past it returns -1
    assert list(st) == [M.OK] * 6 and [int(x) for x in res] == [1, 1, 1, M32, M32, 1]
    _lanes_equal_model(data, 'grow', rows, dev, **lim)
    rows = [(0,), (1,), (2,), (3,), (M32,)]
    res, st = dev.run('table', rows)         # element 0 fits, element 1 has another type, 2 is empty, 3+ is outside
    assert list(st) == [M.OK, M.INDIRECT, M.INDIRECT, M.INDIRECT, M.INDIRECT] and res[0] == 12
    _lanes_equal_model(data, 'table', rows, dev, **lim)
    # out of stack slots with the depth cap far away: recurse's frame is its local + an operand height of 2, and each
    # level starts one slot above its caller's, so 256 slots hold 254 levels
    dev.set_limits(max_depth=100000, stack_slots=256)
    rows = [(0,), (100,), (253,), (254,), (10 ** 6,)] * 8
    res, st = dev.run('recurse', rows)
    for (n,), r, s_ in zip(rows, res, st):
        assert (s_, r) == ((M.OK, n) if n <= 253 else (M.STACK, 0)), (n, s_, r)
    # a budget below one warp's lane state is refused, not exceeded
    dev.set_limits(budget_bytes=4096)
    with pytest.raises(B2gError, match="below one warp's lane state"):
        dev.run('recurse', [(1,)])
    mem = _mem_module()
    d2 = WasmModule(mem, ctx)
    res, st = d2.run('ld28', [(0,), (65532,), (65533,), (0,)])
    assert list(st) == [M.OK, M.OK, M.MEMORY, M.OK]
    d2.close()
    dev.close()


def test_many_globals_get_room_in_the_slots(ctx):
    """the globals sit in each lane's first slots: the default stack_slots grows with them, and a limit that leaves no
    room above them is refused"""
    n = 5000
    glob = [(A.I32, 1, A.i32c(1000 + k)) for k in range(n)]
    get = b'\x23' + A.uleb(n - 1) + b'\x23\x00' + b'\x6a' + A.lget(0) + b'\x6a'
    setget = A.lget(0) + b'\x24' + A.uleb(n - 2) + b'\x23' + A.uleb(n - 2)
    data = A.module([A.Func([A.I32], [A.I32], get, export='get'), A.Func([A.I32], [A.I32], setget, export='setget')],
                    globals_=glob)
    dev = WasmModule(data, ctx)
    assert dev.limits.stack_slots >= n + 8
    rows = [(k,) for k in range(70)]
    _lanes_equal_model(data, 'get', rows, dev)
    _lanes_equal_model(data, 'setget', rows, dev)
    res, st = dev.run('get', rows)
    assert not st.any() and [int(x) for x in res] == [1000 + n - 1 + 1000 + k for k in range(70)]
    for slots in (4096, n + 7):
        with pytest.raises(B2gError, match='stack_slots must be in'):
            dev.set_limits(stack_slots=slots)
    dev.set_limits(stack_slots=n + 8)
    res, st = dev.run('get', rows)
    assert not st.any() and int(res[3]) == 1000 + n - 1 + 1000 + 3
    dev.close()


def test_refusals_name_their_cause(ctx):
    with pytest.raises(B2gError, match='circom 1'):
        WitnessCalculator.new(_wasm('complex-circuit-10000-10000.wasm'), ctx)
    flt = A.module([A.Func([A.I32], [A.I32], A.lget(0) + b'\x45', export='ok'),
                    A.Func([A.I64], [A.I32], A.lget(0) + b'\xb4\xa8', export='f')])
    with pytest.raises(B2gError, match=r'function 1: opcode 0xb4'):
        WasmModule(flt, ctx)
    simd = A.module([A.Func([], [], b'\xfd\x0c' + bytes(16) + b'\x1a', export='v')])
    with pytest.raises(B2gError, match=r'function 0: opcode 0xfd'):
        WasmModule(simd, ctx)
    bulk = A.module([A.Func([A.I32], [], A.lget(0) + A.i32c(0) + A.i32c(1) + b'\xfc\x0b\x00', export='fill')], memory=(1, None))
    with pytest.raises(B2gError, match=r'opcode 0xfc'):
        WasmModule(bulk, ctx)
    imp = A.module([A.Func([], [], b'', export='x')], imports=[('env', 'abort', [A.I32], [])])
    with pytest.raises(B2gError, match=r'env.abort'):
        WasmModule(imp, ctx)
    # a well-formed module without the protocol exports: refused by the witness loader, accepted as a plain module
    with pytest.raises(B2gError, match='does not export the circom 2 function'):
        WitnessCalculator.new(_control_module(), ctx)
    # the exports of a circom 2 module with another field: n32 != 8 and a prime other than r
    for n32, prime in ((4, R), (8, R + 2)):
        with pytest.raises(B2gError, match='getFieldNumLen32|prime'):
            WitnessCalculator.new(_fake_circom(n32, prime), ctx)
    with pytest.raises(B2gError, match='trapped while reporting its field'):
        WitnessCalculator.new(_fake_circom(None, R), ctx)
    assert WitnessCalculator.new(_fake_circom(8, R), ctx).witness_size == 1


def _fake_circom(n32, prime):
    """a module with the circom 2 exports: the prime sits at address 0, readSharedRWMemory(i) reads its word i;
    n32 None: getFieldNumLen32 traps"""
    noop1 = A.Func([A.I32], [], b'', export='init')
    fs = [noop1, A.Func([A.I32, A.I32], [], b'', export='writeSharedRWMemory'),
          A.Func([A.I32, A.I32, A.I32], [], b'', export='setInputSignal'),
          A.Func([], [A.I32], A.i32c(1), export='getWitnessSize'), A.Func([A.I32], [], b'', export='getWitness'),
          A.Func([A.I32], [A.I32], A.lget(0) + A.i32c(2) + b'\x74' + A.memarg(0x28), export='readSharedRWMemory'),
          A.Func([], [A.I32], A.i32c(2), export='getVersion'), A.Func([], [A.I32], A.i32c(n32) if n32 is not None else b'\x00', export='getFieldNumLen32'),
          A.Func([], [], b'', export='getRawPrime'), A.Func([], [A.I32], A.i32c(0), export='getInputSize')]
    return A.module(fs, memory=(1, None), data=[(0, prime.to_bytes(32, 'little'))])


# ------------------------------------------------------------------------------------------------ the fixtures
@pytest.fixture(scope='module')
def calcs(ctx):
    c = {n: WitnessCalculator.new(os.path.join(GOLDEN, n + '.wasm'), ctx) for n in ('mycircuit', 'circuit2')}
    yield c
    for x in c.values():
        x.close()


@pytest.fixture(scope='module')
def models():
    return {n: M.Calculator(_wasm(n + '.wasm')) for n in ('mycircuit', 'circuit2')}


def _r1cs(name):
    return R1CS.from_file(R1CSFile.new(_wasm(name + '.r1cs')))


def _satisfied(r1cs, w):
    for a, b, c in r1cs.constraints:
        ev = [sum(v * w[i] for i, v in lc) % R for lc in (a, b, c)]
        if ev[0] * ev[1] % R != ev[2]:
            return False
    return True


def test_calculator_reads_the_field(calcs):
    for name, size in (('mycircuit', 4), ('circuit2', 132)):
        c = calcs[name]
        assert c.prime == R and c.n64 == 4 and c.n32 == 8 and c.version == 2
        assert c.witness_size == size and c.input_size == 2


def test_fixture_kats(calcs, golden):
    k = golden['witness_kats']
    for wit, inp in zip(k['multiplier'], k['multiplier_inputs']):
        assert calcs['mycircuit'].calculate_witness({'a': int(inp['a']), 'b': int(inp['b'])}) == [int(x) for x in wit]
    w = calcs['circuit2'].calculate_witness({'a': [3], 'b': [11]})
    assert w == [int(x) for x in k['safe_multiplier']] == read_wtns(_wasm('circuit2_witness.wtns'))
    assert calcs['circuit2'].calculate_witness_element([('a', 3), ('b', 11)]) == w


@pytest.mark.parametrize('count', [1, 31, 32, 33, 1024])
@pytest.mark.parametrize('name', ['mycircuit', 'circuit2'])
def test_fixtures_at_many_counts(calcs, models, name, count):
    rng = random.Random(count * 7 + len(name))
    if name == 'mycircuit':
        ins = [(rng.randrange(R), rng.randrange(R)) for _ in range(count)]
    else:
        ins = [(rng.randrange(2, 1 << 64), rng.randrange(2, 1 << 64)) for _ in range(count)]
    wm, st = calcs[name].calculate_witnesses([{'a': a, 'b': b} for a, b in ins])
    assert wm.shape == (count, 4 * calcs[name].witness_size) and not st.any()
    r1cs = _r1cs(name)
    check = range(count) if count <= 64 else rng.sample(range(count), 64)
    for i in check:
        w = fr_from_mont(wm[i])
        a, b = ins[i]
        assert w[:4] == [1, a * b % R, a, b] and _satisfied(r1cs, w)
    for i in sorted({0, count - 1, count // 2}):     # whole witnesses against the model
        ms, mw = models[name].calculate([('a', [ins[i][0]]), ('b', [ins[i][1]])])
        assert ms == M.OK and fr_from_mont(wm[i]) == mw


def test_chunking_does_not_change_results(ctx, calcs):
    rng = random.Random(5)
    ins = [{'a': rng.randrange(2, 1 << 64), 'b': rng.randrange(2, 1 << 64)} for _ in range(100)]
    ins[37]['a'] = 1                                             # a failing lane in the middle of a chunk
    whole, st0 = calcs['circuit2'].calculate_witnesses(ins)
    small = WitnessCalculator.new(os.path.join(GOLDEN, 'circuit2.wasm'), ctx)
    lim = small.limits
    per_lane = lim.max_pages * 65536 + lim.stack_slots * 8 + lim.max_depth * 8 + 2 * 32 + 132 * 32 + 4
    small.set_limits(budget_bytes=per_lane * 40)                # chunks of 32 lanes: four of them
    parts, st1 = small.calculate_witnesses(ins)
    assert np.array_equal(whole, parts) and np.array_equal(st0, st1)
    assert st0[37] == M.EXCEPTION + 4 and not np.delete(st0, 37).any() and not whole[37].any()
    small.close()


def test_inputs_at_and_above_r_and_negative(calcs, models):
    wm, st = calcs['mycircuit'].calculate_witnesses([{'a': R + 3, 'b': -11}, {'a': 3, 'b': R - 11}, {'a': -1, 'b': 2 * R}])
    assert not st.any()
    w = [fr_from_mont(x) for x in wm]
    assert w[0] == w[1] == [1, 3 * (R - 11) % R, 3, R - 11] and w[2] == [1, 0, R - 1, 0]
    assert models['mycircuit'].calculate([('a', [R + 3]), ('b', [-11])])[1] == w[0]


def test_circuit2_failing_lanes_leave_their_neighbours_alone(calcs, models):
    rng = random.Random(11)
    ins = [(rng.randrange(2, 1 << 64), rng.randrange(2, 1 << 64)) for _ in range(64)]
    bad = {3: (1 << 64, 5), 4: (1, 5), 31: (5, 1), 32: (R - 1, 7), 40: (-5, 9), 63: ((1 << 64) + 2, 3)}
    ins = [bad.get(i, x) for i, x in enumerate(ins)]
    wm, st = calcs['circuit2'].calculate_witnesses([{'a': a, 'b': b} for a, b in ins])
    for i, (a, b) in enumerate(ins):
        if i in bad:
            ms, _ = models['circuit2'].calculate([('a', [a]), ('b', [b])])
            assert ms == M.EXCEPTION + 4 and st[i] == ms and not wm[i].any()
        else:
            assert st[i] == 0 and fr_from_mont(wm[i])[:4] == [1, a * b % R, a, b]
    with pytest.raises(WitnessError, match='Assert Failed'):
        calcs['circuit2'].calculate_witness({'a': 1, 'b': 3})


# ------------------------------------------------------------------------------------------------ end to end
def test_builder_with_the_wasm_proves_and_verifies(ctx):
    """tests/groth16.rs:75-105 with circuit2.wasm in place of the .wtns: build() computes the witness on the GPU"""
    cfg = CircomConfig.new(os.path.join(GOLDEN, 'circuit2.wasm'), os.path.join(GOLDEN, 'circuit2.r1cs'))
    builder = CircomBuilder.new(cfg)
    builder.push_input('a', 3)
    builder.push_input('b', 11)
    circom = builder.setup()
    rng = random.Random(2024)
    pk = Groth16.generate_random_parameters_with_reduction(circom.to_circuit(), rng, ctx)
    circom = builder.build()
    assert circom.witness == read_wtns(_wasm('circuit2_witness.wtns'))
    inputs = circom.get_public_inputs()
    assert inputs == [33]
    cm = circom.to_circuit().matrices()
    proof = Groth16.prove(pk, cm, fr_to_mont(circom.witness), rng, ctx)
    assert Groth16.verify(pk, inputs, proof)
    assert not Groth16.verify(pk, [34], proof)
    # a batch of 256 GPU witnesses proved in one pass and verified in one pass
    calc = cfg.wasm
    ab = [(rng.randrange(2, 1 << 64), rng.randrange(2, 1 << 64)) for _ in range(256)]
    wm, st = calc.calculate_witnesses([{'a': a, 'b': b} for a, b in ab])
    assert not st.any()
    proofs = Groth16.create_proofs(pk, [(rng.randrange(1, R), rng.randrange(1, R)) for _ in ab], cm, wm, ctx)
    pubs = [[a * b % R] for a, b in ab]
    assert Groth16.verify_many(pk, pubs, proofs, ctx) == [True] * 256
    release(pk); release(cm)


def test_cpp_mirror_witnesses_equal_python(calcs, tmp_path):
    """B2G_WITNESS=circuit2.wasm groth16_bench circuit2.r1cs a=.. b=.. count: the C++ WitnessCalculator's witnesses, proved
    and verified there, equal the Python ones word for word"""
    out = tmp_path / 'w.bin'
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    env = dict(os.environ, B2G_WITNESS=os.path.join(GOLDEN, 'circuit2.wasm'), B2G_WITNESS_OUT=str(out))
    p = subprocess.run([exe, os.path.join(GOLDEN, 'circuit2.r1cs'), 'a=3', 'b=11', '40'], env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert 'verified 40/40' in p.stdout, p.stdout
    got = np.fromfile(out, dtype=np.uint64).reshape(40, -1)
    want, st = calcs['circuit2'].calculate_witnesses([{'a': 3, 'b': 11}] * 40)
    assert not st.any() and np.array_equal(got, want)
