"""Plain-Python model of the circom 2 witness calculator: a WebAssembly decoder and interpreter for the integer subset of
the MVP, and the circom 2 calling protocol on top of it.

It works on the raw module bytes and shares nothing with the library's translator (csrc/wasm.cu): blocks are matched by
a scan of each body and branches walk a runtime label stack, the way the specification describes them.  It is the
yardstick the device interpreter is tested against, one witness at a time.

Lane statuses (the same numbers b2g_witness_calculate writes):
    0 ok, 1 unreachable, 2 memory access out of bounds, 3 integer division by zero, 4 integer overflow,
    5 call stack exhausted, 6 fuel exhausted, 7 bad call_indirect, 8 getWitnessSize after the inputs disagrees with
    the size the module reported before init, 0x100 + c the circuit called exceptionHandler(c)
"""
from __future__ import annotations

R_MOD = 21888242871839275222246405745257275088548364400416034343698204186575808495617
PAGE = 65536
M32, M64 = (1 << 32) - 1, (1 << 64) - 1

OK, UNREACHABLE, MEMORY, DIV_ZERO, OVERFLOW, STACK, FUEL, INDIRECT, PROTOCOL = range(9)
EXCEPTION = 0x100

RUNTIME_IMPORTS = {'exceptionHandler': (1, 0), 'printErrorMessage': (0, 0), 'writeBufferMessage': (0, 0),
                   'showSharedRWMemory': (0, 0)}
PROTOCOL_EXPORTS = ['getFieldNumLen32', 'getRawPrime', 'readSharedRWMemory', 'writeSharedRWMemory', 'init',
                    'setInputSignal', 'getWitnessSize', 'getWitness', 'getInputSize', 'getVersion']


class Refused(ValueError):
    """the module is outside what the calculator runs"""


class Trap(Exception):
    def __init__(self, status):
        super().__init__(status)
        self.status = status


def fnv1a64(name: str) -> int:
    h = 0xcbf29ce484222325
    for b in name.encode():
        h = ((h ^ b) * 0x100000001b3) & M64
    return h


# ----------------------------------------------------------------------------------------------------------- decoding
class _Reader:
    def __init__(self, b, pos=0, end=None):
        self.b, self.p, self.end = b, pos, len(b) if end is None else end

    def byte(self):
        if self.p >= self.end:
            raise Refused("truncated module")
        v = self.b[self.p]
        self.p += 1
        return v

    def uleb(self):
        r = s = 0
        while True:
            v = self.byte()
            r |= (v & 0x7f) << s
            s += 7
            if not v & 0x80:
                return r

    def sleb(self, bits):
        r = s = 0
        while True:
            v = self.byte()
            r |= (v & 0x7f) << s
            s += 7
            if not v & 0x80:
                if v & 0x40:
                    r -= 1 << s
                return r & ((1 << bits) - 1)

    def name(self):
        n = self.uleb()
        v = bytes(self.b[self.p:self.p + n])
        self.p += n
        return v.decode()

    def limits(self):
        flag = self.byte()
        lo = self.uleb()
        return lo, (self.uleb() if flag & 1 else None)


def _const_expr(r):
    op = r.byte()
    if op == 0x41:
        v = ('i32', r.sleb(32))
    elif op == 0x42:
        v = ('i64', r.sleb(64))
    elif op == 0x23:
        v = ('global', r.uleb())
    else:
        raise Refused(f"constant expression opcode 0x{op:02x} is not supported")
    if r.byte() != 0x0b:
        raise Refused("constant expression is not a single constant")
    return v


class Module:
    def __init__(self, data: bytes, protocol: bool = True):
        if data[:4] != b'\0asm' or data[4:8] != b'\x01\0\0\0':
            raise Refused("not a WebAssembly 1 binary")
        self.types, self.imports, self.func_types, self.codes = [], [], [], []
        self.table, self.mem, self.globals, self.exports, self.elems, self.datas = None, None, [], {}, [], []
        self.start = None
        r = _Reader(data, 8)
        while r.p < len(data):
            sid, size = r.byte(), r.uleb()
            s = _Reader(data, r.p, r.p + size)
            r.p += size
            if sid == 1:
                for _ in range(s.uleb()):
                    if s.byte() != 0x60:
                        raise Refused("bad function type")
                    ps = [s.byte() for _ in range(s.uleb())]
                    rs = [s.byte() for _ in range(s.uleb())]
                    for t in ps + rs:
                        if t not in (0x7f, 0x7e):
                            raise Refused(f"value type 0x{t:02x} in a function type is not supported")
                    self.types.append((tuple(ps), tuple(rs)))
            elif sid == 2:
                for _ in range(s.uleb()):
                    mod, nm, kind = s.name(), s.name(), s.byte()
                    if kind != 0:
                        raise Refused(f"import {mod}.{nm} is not a function (circom 1 modules import env.memory)")
                    if mod != 'runtime' or nm not in RUNTIME_IMPORTS:
                        raise Refused(f"import {mod}.{nm} is not one of the circom 2 runtime functions")
                    t = s.uleb()
                    self.imports.append((nm, t))
            elif sid == 3:
                self.func_types += [s.uleb() for _ in range(s.uleb())]
            elif sid == 4:
                for _ in range(s.uleb()):
                    if s.byte() != 0x70:
                        raise Refused("table of a type other than funcref")
                    self.table = s.limits()
            elif sid == 5:
                for _ in range(s.uleb()):
                    self.mem = s.limits()
            elif sid == 6:
                for _ in range(s.uleb()):
                    t, mut = s.byte(), s.byte()
                    if t not in (0x7f, 0x7e):
                        raise Refused(f"global of value type 0x{t:02x} is not supported")
                    self.globals.append((t, mut, _const_expr(s)))
            elif sid == 7:
                for _ in range(s.uleb()):
                    nm, kind, idx = s.name(), s.byte(), s.uleb()
                    self.exports[nm] = (kind, idx)
            elif sid == 8:
                self.start = s.uleb()
            elif sid == 9:
                for _ in range(s.uleb()):
                    if s.uleb() != 0:
                        raise Refused("element segment other than an active one of table 0")
                    off = _const_expr(s)
                    self.elems.append((off, [s.uleb() for _ in range(s.uleb())]))
            elif sid == 10:
                for _ in range(s.uleb()):
                    size = s.uleb()
                    body = _Reader(data, s.p, s.p + size)
                    s.p += size
                    locs = []
                    for _ in range(body.uleb()):
                        n, t = body.uleb(), body.byte()
                        if t not in (0x7f, 0x7e):
                            raise Refused(f"function {len(self.imports) + len(self.codes)}: local of value type 0x{t:02x}")
                        locs += [t] * n
                    self.codes.append((locs, body.p, body.end))
            elif sid == 11:
                for _ in range(s.uleb()):
                    if s.uleb() != 0:
                        raise Refused("data segment other than an active one of memory 0")
                    off = _const_expr(s)
                    n = s.uleb()
                    self.datas.append((off, bytes(data[s.p:s.p + n])))
                    s.p += n
            elif sid == 12:
                raise Refused("bulk-memory data count section")
        self.data = data
        if len(self.codes) != len(self.func_types):
            raise Refused("function and code sections disagree")
        if self.mem is None:
            if protocol:
                raise Refused("the module defines no memory")
            self.mem = (0, 0)
        self.bodies = [None] * len(self.codes)
        for nm in PROTOCOL_EXPORTS if protocol else []:
            if nm not in self.exports or self.exports[nm][0] != 0:
                raise Refused(f"the module does not export the circom 2 function {nm}")

    def ftype(self, f):
        return self.types[self.imports[f][1] if f < len(self.imports) else self.func_types[f - len(self.imports)]]

    def body(self, k):
        """the decoded body of defined function k: a list of (op, imm) and, for block openers, their else/end positions"""
        if self.bodies[k] is None:
            self.bodies[k] = _decode_body(self, k)
        return self.bodies[k]


_LOAD = {0x28: (4, 32, False), 0x29: (8, 64, False), 0x2c: (1, 32, True), 0x2d: (1, 32, False), 0x2e: (2, 32, True),
         0x2f: (2, 32, False), 0x30: (1, 64, True), 0x31: (1, 64, False), 0x32: (2, 64, True), 0x33: (2, 64, False),
         0x34: (4, 64, True), 0x35: (4, 64, False)}
_STORE = {0x36: 4, 0x37: 8, 0x3a: 1, 0x3b: 2, 0x3c: 1, 0x3d: 2, 0x3e: 4}
_PLAIN = set(range(0x45, 0x5b)) | set(range(0x67, 0x8b)) | {0xa7, 0xac, 0xad} | set(range(0xc0, 0xc5)) | {0x00, 0x01, 0x0f, 0x1a, 0x1b}


def _decode_body(m, k):
    fi = len(m.imports) + k
    _, start, end = m.codes[k]
    r = _Reader(m.data, start, end)
    code, opens = [], []
    while r.p < end:
        op = r.byte()
        if op in (0x02, 0x03, 0x04):
            bt = r.byte()
            if bt == 0x40:
                arity = 0
            elif bt in (0x7f, 0x7e):
                arity = 1
            else:
                raise Refused(f"function {fi}: block type 0x{bt:02x} is not supported")
            opens.append(len(code))
            code.append([op, arity, None, None])     # op, arity, else pc, end pc
        elif op == 0x05:
            code[opens[-1]][2] = len(code)
            code.append([op])
        elif op == 0x0b:
            if opens:
                code[opens.pop()][3] = len(code)
            code.append([op])
        elif op in (0x0c, 0x0d, 0x10, 0x20, 0x21, 0x22, 0x23, 0x24):
            code.append([op, r.uleb()])
        elif op == 0x0e:
            tab = [r.uleb() for _ in range(r.uleb())]
            code.append([op, tab, r.uleb()])
        elif op == 0x11:
            t = r.uleb()
            if r.byte() != 0:
                raise Refused(f"function {fi}: call_indirect on a table other than 0")
            code.append([op, t])
        elif op in _LOAD or op in _STORE:
            r.uleb()
            code.append([op, r.uleb()])
        elif op in (0x3f, 0x40):
            if r.byte() != 0:
                raise Refused(f"function {fi}: memory index other than 0")
            code.append([op])
        elif op == 0x41:
            code.append([op, r.sleb(32)])
        elif op == 0x42:
            code.append([op, r.sleb(64)])
        elif op in _PLAIN:
            code.append([op])
        else:
            raise Refused(f"function {fi}: opcode 0x{op:02x} is not in the integer subset")
    return code


# ----------------------------------------------------------------------------------------------------------- execution
def _s32(v):
    return v - (1 << 32) if v & 0x80000000 else v


def _s64(v):
    return v - (1 << 64) if v >> 63 else v


def _clz(v, w):
    return w - v.bit_length()


def _ctz(v, w):
    return w if v == 0 else (v & -v).bit_length() - 1


def _tdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def _binop(op, a, b):
    """i32 ops 0x6a-0x78 and i64 ops 0x7c-0x8a; a, b unsigned"""
    w, M = (32, M32) if op <= 0x78 else (64, M64)
    o = op - (0x6a if op <= 0x78 else 0x7c)
    s = _s32 if w == 32 else _s64
    if o == 0:
        return (a + b) & M
    if o == 1:
        return (a - b) & M
    if o == 2:
        return (a * b) & M
    if o in (3, 4, 5, 6):
        if b == 0:
            raise Trap(DIV_ZERO)
        if o == 3:
            if s(a) == -(1 << (w - 1)) and s(b) == -1:
                raise Trap(OVERFLOW)
            return _tdiv(s(a), s(b)) & M
        if o == 4:
            return a // b
        if o == 5:
            return (s(a) - _tdiv(s(a), s(b)) * s(b)) & M
        return a % b
    if o == 7:
        return a & b
    if o == 8:
        return a | b
    if o == 9:
        return a ^ b
    k = b % w
    if o == 10:
        return (a << k) & M
    if o == 11:
        return (s(a) >> k) & M
    if o == 12:
        return a >> k
    if o == 13:
        return ((a << k) | (a >> (w - k))) & M
    return ((a >> k) | (a << (w - k))) & M


def _cmp(op, a, b):
    s = _s32 if op <= 0x4f else _s64
    o = op - (0x46 if op <= 0x4f else 0x51)
    return int([a == b, a != b, s(a) < s(b), a < b, s(a) > s(b), a > b, s(a) <= s(b), a <= b, s(a) >= s(b), a >= b][o])


def _sext(v, bits, M):
    v &= (1 << bits) - 1
    return (v - (1 << bits) if v >> (bits - 1) else v) & M


class Instance:
    """one fresh instantiation: memory from the data segments, globals from their initialisers.

    trace: None (the default) or a dict that collects, per defined function k, the set of pcs (indices into
    Module.body(k)) this instance executes; coverage tests pass one in, other callers pay nothing for it."""

    def __init__(self, m: Module, max_pages=None, max_depth=1024, fuel=None, trace=None):
        self.m = m
        self.trace = trace
        lo, hi = m.mem
        self.max_pages = max_pages if max_pages is not None else (hi if hi is not None else 65536)
        if hi is not None:
            self.max_pages = min(self.max_pages, hi)
        self.mem = bytearray(lo * PAGE)
        self.max_depth, self.fuel = max_depth, fuel
        self.globals = []
        for t, _, init in m.globals:
            self.globals.append(self.globals[init[1]] if init[0] == 'global' else init[1])
        self.table = [None] * (m.table[0] if m.table else 0)
        for off, fs in m.elems:
            o = self._const(off)
            if o + len(fs) > len(self.table):
                raise Refused("element segment outside the table")
            self.table[o:o + len(fs)] = fs
        for off, b in m.datas:
            o = self._const(off)
            if o + len(b) > len(self.mem):
                raise Refused("data segment outside the memory")
            self.mem[o:o + len(b)] = b
        self.depth = 0

    def _const(self, e):
        return self.globals[e[1]] if e[0] == 'global' else e[1]

    def call(self, name, *args):
        return self.invoke(self.m.exports[name][1], list(args))

    def invoke(self, f, args):
        m = self.m
        ps, rs = m.ftype(f)
        if f < len(m.imports):
            nm = m.imports[f][0]
            if nm == 'exceptionHandler':
                raise Trap(EXCEPTION + (args[0] & M32))
            return []
        self.depth += 1
        if self.depth > self.max_depth:
            raise Trap(STACK)
        try:
            return self._run(f, args)
        finally:
            self.depth -= 1

    def _tick(self):
        if self.fuel is not None:
            self.fuel -= 1
            if self.fuel < 0:
                raise Trap(FUEL)

    def _addr(self, base, off, n):
        a = base + off
        if a + n > len(self.mem):
            raise Trap(MEMORY)
        return a

    def _run(self, f, args):
        m = self.m
        k = f - len(m.imports)
        locs = args + [0] * len(m.codes[k][0])
        code = m.body(k)
        nres = len(m.ftype(f)[1])
        st, labels = [], []        # labels: (pc to go to on a branch, arity on a branch, height, is loop)
        pc, n = 0, len(code)
        tr = self.trace.setdefault(k, set()) if self.trace is not None else None
        while pc < n:
            if tr is not None:
                tr.add(pc)
            ins = code[pc]
            op = ins[0]
            pc += 1
            self._tick()
            if op == 0x20:
                st.append(locs[ins[1]])
            elif op == 0x21:
                locs[ins[1]] = st.pop()
            elif op == 0x22:
                locs[ins[1]] = st[-1]
            elif op == 0x41 or op == 0x42:
                st.append(ins[1])
            elif 0x6a <= op <= 0x78 or 0x7c <= op <= 0x8a:
                b = st.pop()
                st.append(_binop(op, st.pop(), b))
            elif op in _LOAD:
                nb, w, sg = _LOAD[op]
                a = self._addr(st.pop(), ins[1], nb)
                v = int.from_bytes(self.mem[a:a + nb], 'little')
                st.append(_sext(v, 8 * nb, (1 << w) - 1) if sg else v)
            elif op in _STORE:
                nb = _STORE[op]
                v = st.pop()
                a = self._addr(st.pop(), ins[1], nb)
                self.mem[a:a + nb] = (v & ((1 << (8 * nb)) - 1)).to_bytes(nb, 'little')
            elif op == 0x02 or op == 0x03:
                end = ins[3]
                labels.append((pc - 1, 0, len(st), True) if op == 0x03 else (end + 1, ins[1], len(st), False))
            elif op == 0x04:
                c = st.pop()
                labels.append((ins[3] + 1, ins[1], len(st), False))
                if not c:
                    if ins[2] is not None:
                        pc = ins[2] + 1
                    else:
                        pc = ins[3] + 1
                        labels.pop()
            elif op == 0x05:          # reached the else at the end of a then-arm: leave the if
                pc = labels.pop()[0]
            elif op == 0x0b:
                if labels:
                    labels.pop()
                else:
                    break
            elif op == 0x0c or op == 0x0d or op == 0x0e:
                if op == 0x0d:
                    if not st.pop():
                        continue
                    depth = ins[1]
                elif op == 0x0e:
                    i = st.pop()
                    depth = ins[1][i] if i < len(ins[1]) else ins[2]
                else:
                    depth = ins[1]
                if depth == len(labels):
                    break                                          # a branch to the function's own block returns
                target, arity, h, _ = labels[-1 - depth]
                vals = st[len(st) - arity:] if arity else []
                del st[h:]
                st += vals
                del labels[len(labels) - 1 - depth:]
                pc = target
            elif op == 0x0f:
                break
            elif op == 0x10 or op == 0x11:
                if op == 0x11:
                    i = st.pop()
                    if i >= len(self.table) or self.table[i] is None:
                        raise Trap(INDIRECT)
                    g = self.table[i]
                    if m.ftype(g) != m.types[ins[1]]:
                        raise Trap(INDIRECT)
                else:
                    g = ins[1]
                np_ = len(m.ftype(g)[0])
                a = st[len(st) - np_:] if np_ else []
                del st[len(st) - np_:]
                st += self.invoke(g, a)
            elif op == 0x23:
                st.append(self.globals[ins[1]])
            elif op == 0x24:
                self.globals[ins[1]] = st.pop()
            elif 0x46 <= op <= 0x4f or 0x51 <= op <= 0x5a:
                b = st.pop()
                st.append(_cmp(op, st.pop(), b))
            elif op == 0x45 or op == 0x50:
                st.append(int(st.pop() == 0))
            elif op == 0x1a:
                st.pop()
            elif op == 0x1b:
                c, b = st.pop(), st.pop()
                a = st.pop()
                st.append(a if c else b)
            elif op == 0x01:
                pass
            elif op == 0x00:
                raise Trap(UNREACHABLE)
            elif op == 0x3f:
                st.append(len(self.mem) // PAGE)
            elif op == 0x40:
                d = st.pop()
                old = len(self.mem) // PAGE
                if old + d > self.max_pages:
                    st.append(M32)
                else:
                    self.mem.extend(bytes(d * PAGE))
                    st.append(old)
            elif op in (0x67, 0x68, 0x69, 0x79, 0x7a, 0x7b):
                w = 32 if op <= 0x69 else 64
                v = st.pop()
                o = op - (0x67 if w == 32 else 0x79)
                st.append(_clz(v, w) if o == 0 else _ctz(v, w) if o == 1 else bin(v).count('1'))
            elif op == 0xa7:
                st.append(st.pop() & M32)
            elif op == 0xac:
                st.append(_sext(st.pop(), 32, M64))
            elif op == 0xad:
                st.append(st.pop() & M32)
            elif op == 0xc0:
                st.append(_sext(st.pop(), 8, M32))
            elif op == 0xc1:
                st.append(_sext(st.pop(), 16, M32))
            elif op == 0xc2:
                st.append(_sext(st.pop(), 8, M64))
            elif op == 0xc3:
                st.append(_sext(st.pop(), 16, M64))
            elif op == 0xc4:
                st.append(_sext(st.pop(), 32, M64))
            else:
                raise AssertionError(f"opcode 0x{op:02x}")
        return st[len(st) - nres:] if nres else []


# ----------------------------------------------------------------------------------------------------------- protocol
class Calculator:
    """the circom 2 protocol over one module; every witness runs on a fresh instance"""

    def __init__(self, data: bytes, **limits):
        self.m = Module(data)
        self.limits = limits
        inst = Instance(self.m, **limits)
        self.version = inst.call('getVersion')[0]
        self.n32 = inst.call('getFieldNumLen32')[0]
        inst.call('getRawPrime')
        self.prime = sum(inst.call('readSharedRWMemory', j)[0] << (32 * j) for j in range(self.n32))
        self.witness_size = inst.call('getWitnessSize')[0]
        self.input_size = inst.call('getInputSize')[0]
        if self.prime != R_MOD:
            raise Refused(f"the circuit's prime {self.prime:#x} is not BN254's scalar field modulus")
        if self.n32 != 8:
            raise Refused(f"getFieldNumLen32 = {self.n32}, expected 8")

    def calculate(self, inputs, sanity_check=False):
        """inputs: [(name, [values])]; returns (status, witness): witness is the list of ints when status is 0"""
        inst = Instance(self.m, **self.limits)
        try:
            inst.call('init', int(bool(sanity_check)))
            for name, values in inputs:
                h = fnv1a64(name)
                for i, v in enumerate(values):
                    v = int(v) % R_MOD
                    for j in range(self.n32):
                        inst.call('writeSharedRWMemory', j, (v >> (32 * j)) & M32)
                    inst.call('setInputSignal', h >> 32, h & M32, i)
            n = inst.call('getWitnessSize')[0]
            if n != self.witness_size:         # the witness would not have the rows the caller allocated
                return PROTOCOL, None
            w = []
            for i in range(n):
                inst.call('getWitness', i)
                w.append(sum(inst.call('readSharedRWMemory', j)[0] << (32 * j) for j in range(self.n32)))
            return OK, w
        except Trap as t:
            return t.status, None


def run_function(data: bytes, name: str, args, **limits):
    """calls one export of a module (a hand-built one need not follow the protocol) on a fresh instance:
    (status, results)"""
    inst = Instance(Module(data, protocol=False), **limits)
    try:
        return OK, inst.call(name, *args)
    except Trap as t:
        return t.status, None
