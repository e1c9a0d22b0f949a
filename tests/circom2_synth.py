"""Hand-built circom 2 modules for the witness driver (b2g_witness_calculate, mode 1 of csrc/wasm.cu).

No circom compiler is needed: `Synth` writes, with tests/wasm_asm.py, a module that follows the calling protocol the
driver (and ark-circom's WitnessCalculator) uses, over input signals of any sizes and a witness of any size:

- memory: the 8 shared words at 0, r at 32, three cells (init ran, values set, fault mode) at 64, the signal table at
  128 (FNV-1a msb, lsb, first element, size: four words per signal), one "set" flag per input element, then the wires
  (8 words each);
- setInputSignal(msb, lsb, i) looks the hash up and stores the shared words in wire 1 + first + i.  It calls
  runtime.exceptionHandler with circom 2's codes: 1 for an unknown hash, 6 for i >= size, 3 for an element set twice
  and 2 for more values than getInputSize;
- when the last value is set (in init when there are none) the module computes its witness: wire 0 is 1, wires 1.. are
  the input elements in table order, and every later wire k is w[k - 1] + w[b(k)] mod r (b(k) in `pattern`), by one
  8-limb add-with-carry and conditional subtraction of r written with i64 operations.

The expected witness (`expected`) is plain integer arithmetic and never reads the module.

Fault switches: `protocol_fault` makes getWitnessSize return N + 1 once init has run (B2G_WASM_PROTOCOL);
`claimed_size` makes it report another size outright; `input_size` overrides getInputSize.  `mode` names an input
signal of size 1 whose value picks a per-lane fault (`MODES`), so one call can end each lane differently: 1, 2, 3 and 6
bend every later setInputSignal into that exception, 4 fails an assert, 8 reports N + 1 wires and 9 loops forever.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Sequence, Tuple

import wasm_asm as A
from wasm_model import EXCEPTION, FUEL, M32, OK, PROTOCOL, R_MOD, fnv1a64

MODES = {0: OK, 1: EXCEPTION + 1, 2: EXCEPTION + 2, 3: EXCEPTION + 3, 4: EXCEPTION + 4, 6: EXCEPTION + 6, 8: PROTOCOL,
         9: FUEL}
MULT = 0x9E3779B1

SHARED, RADDR, CELL_INIT, CELL_COUNT, CELL_MODE, TAB = 0, 32, 64, 68, 72, 128
EXC, COMPUTE, ADD = 0, 5, 4           # function indices: the first import, then the defined functions below


def pattern(k: int) -> int:
    """the second operand of wire k (the first is k - 1)"""
    return (((k * MULT) & M32) >> 7) % k


# ------------------------------------------------------------------------------------------------ opcodes
def _op(*b):
    return bytes(b)


def c32(v):
    return A.i32c(v & M32)


def lg(i):
    return A.lget(i)


def ls(i):
    return b'\x21' + A.uleb(i)


def lt(i):
    return b'\x22' + A.uleb(i)


def ld32(off=0):
    return A.memarg(0x28, off)


def st32(off=0):
    return A.memarg(0x36, off)


def ld64u32(off=0):
    return A.memarg(0x35, off)


def st64_32(off=0):
    return A.memarg(0x3e, off)


def call(f):
    return b'\x10' + A.uleb(f)


IF, ELSE, END, BLOCK, LOOP, RETURN = b'\x04\x40', b'\x05', b'\x0b', b'\x02\x40', b'\x03\x40', b'\x0f'
EQ, GE_U, ADD32, SUB32, MUL32, REMU, AND32, XOR32, SHL, SHRU = (_op(x) for x in (0x46, 0x4f, 0x6a, 0x6b, 0x6c, 0x70, 0x71,
                                                                                0x73, 0x74, 0x76))
I64ADD, I64SUB, I64SHRU, I64EQZ = _op(0x7c), _op(0x7d), _op(0x88), _op(0x50)


def br(d):
    return b'\x0c' + A.uleb(d)


def br_if(d):
    return b'\x0d' + A.uleb(d)


def throw(code):
    return c32(code) + call(EXC) + RETURN


# ------------------------------------------------------------------------------------------------ the module
class Synth:
    def __init__(self, signals: Sequence[Tuple[str, int]], n_wit: Optional[int] = None, mode: Optional[str] = None,
                 input_size: Optional[int] = None, protocol_fault: bool = False, claimed_size: Optional[int] = None):
        self.signals = [(str(n), int(s)) for n, s in signals]
        names = [n for n, _ in self.signals]
        assert len(set(names)) == len(names) and all(s >= 1 for _, s in self.signals)
        self.total = sum(s for _, s in self.signals)
        self.first = {}
        off = 0
        for n, s in self.signals:
            self.first[n] = off
            off += s
        self.n_wit = 1 + self.total if n_wit is None else int(n_wit)
        assert self.n_wit >= 1 + self.total
        self.input_size = self.total if input_size is None else int(input_size)
        self.mode = mode
        if mode is not None:
            assert dict(self.signals)[mode] == 1
        self.protocol_fault, self.claimed_size = protocol_fault, claimed_size
        self.setf = (TAB + 16 * len(self.signals) + 31) // 32 * 32
        self.wires = (self.setf + 4 * self.total + 31) // 32 * 32
        self.pages = max(1, (self.wires + 32 * self.n_wit + 65535) // 65536)
        self.wasm = self._module()

    # -------------------------------------------------------------------------------------------- expectations
    def expected(self, inputs: Dict[str, Sequence[int]]) -> List[int]:
        """the witness for inputs {name: [values]} (any order, any integers; reduced mod r as the host does)"""
        w = [1]
        for n, s in self.signals:
            v = inputs[n]
            v = [v] if isinstance(v, (int, str)) else list(v)
            assert len(v) == s
            w += [int(x) % R_MOD for x in v]
        for k in range(len(w), self.n_wit):
            w.append((w[k - 1] + w[pattern(k)]) % R_MOD)
        return w

    def expected_status(self, inputs: Dict[str, Sequence[int]]) -> int:
        if self.mode is not None:
            m = inputs[self.mode]
            m = int(m if isinstance(m, (int, str)) else list(m)[0]) % R_MOD
            if m in MODES and m != 0:
                return MODES[m]
        if self.input_size < self.total:
            return EXCEPTION + 2
        if self.protocol_fault:
            return PROTOCOL
        return OK

    def r1cs(self, n_public: int = 0) -> bytes:
        """the circuit as a .r1cs: (w[k-1] + w[b(k)]) * 1 = w[k] for every computed wire; the first n_public input
        elements are its public inputs"""
        cons = []
        for k in range(1 + self.total, self.n_wit):
            a, b = k - 1, pattern(k)
            lin = [(a, 2)] if a == b else [(a, 1), (b, 1)]
            cons.append((lin, [(0, 1)], [(k, 1)]))

        def lc(terms):
            return struct.pack('<I', len(terms)) + b''.join(struct.pack('<I', w) + c.to_bytes(32, 'little') for w, c in terms)
        hdr = struct.pack('<I', 32) + R_MOD.to_bytes(32, 'little') + struct.pack(
            '<IIIIQI', self.n_wit, 0, n_public, self.total - n_public, self.n_wit, len(cons))
        body = b''.join(lc(a) + lc(b) + lc(c) for a, b, c in cons)
        labels = struct.pack('<%dQ' % self.n_wit, *range(self.n_wit))
        out = b'r1cs' + struct.pack('<II', 1, 3)
        for t, s in ((1, hdr), (2, body), (3, labels)):
            out += struct.pack('<IQ', t, len(s)) + s
        return out

    # -------------------------------------------------------------------------------------------- code
    def _add(self):
        """add(dst, a, b): w[dst] = w[a] + w[b] mod r, byte addresses; locals 3 carry, 4 sum, 5 borrow, 6..13 limbs"""
        c, t, bw = 3, 4, 5
        body = b''
        for j in range(8):
            body += (lg(0) + lg(1) + ld64u32(4 * j) + lg(2) + ld64u32(4 * j) + I64ADD + lg(c) + I64ADD + lt(t) +
                     st64_32(4 * j) + lg(t) + A.i64c(32) + I64SHRU + ls(c))
        for j in range(8):
            rj = (R_MOD >> (32 * j)) & M32
            body += lg(0) + ld64u32(4 * j) + A.i64c(rj) + I64SUB + lg(bw) + I64SUB + lt(6 + j) + A.i64c(63) + I64SHRU + ls(bw)
        body += lg(bw) + I64EQZ + IF
        for j in range(8):
            body += lg(0) + lg(6 + j) + st64_32(4 * j)
        body += END
        return A.Func([A.I32] * 3, [], body, locals_=[A.I64] * 11)

    def _mode_is(self, m):
        return c32(CELL_MODE) + ld32() + c32(m) + EQ + IF

    def _compute(self):
        W = self.wires
        body = c32(W) + c32(1) + st32()
        if self.mode is not None:
            body += self._mode_is(4) + throw(4) + END
            body += self._mode_is(9) + LOOP + br(0) + END + END
        addr = lambda e: e + c32(5) + SHL + c32(W) + ADD32        # noqa: E731
        body += c32(1 + self.total) + ls(0) + BLOCK + LOOP
        body += lg(0) + c32(self.n_wit) + GE_U + br_if(1)
        body += addr(lg(0)) + addr(lg(0) + c32(1) + SUB32)
        body += addr(lg(0) + c32(MULT) + MUL32 + c32(7) + SHRU + lg(0) + REMU)
        body += call(ADD) + lg(0) + c32(1) + ADD32 + ls(0) + br(0) + END + END
        return A.Func([], [], body, locals_=[A.I32])

    def _set_input(self):
        s, e, p = 3, 4, 5
        body = b''
        if self.mode is not None:
            h = fnv1a64(self.mode)
            body += self._mode_is(1) + lg(0) + c32(1 << 31) + XOR32 + ls(0) + END
            body += self._mode_is(6) + lg(2) + c32(1 << 20) + ADD32 + ls(2) + END
            body += self._mode_is(3) + c32(h >> 32) + ls(0) + c32(h & M32) + ls(1) + c32(0) + ls(2) + END
            body += self._mode_is(2) + c32(CELL_COUNT) + c32(self.input_size) + st32() + END
        body += BLOCK + LOOP
        body += lg(s) + c32(len(self.signals)) + GE_U + IF + throw(1) + END
        body += lg(s) + c32(4) + SHL + c32(TAB) + ADD32 + ls(p)
        body += lg(p) + ld32(0) + lg(0) + EQ + lg(p) + ld32(4) + lg(1) + EQ + AND32 + br_if(1)
        body += lg(s) + c32(1) + ADD32 + ls(s) + br(0) + END + END
        body += lg(2) + lg(p) + ld32(12) + GE_U + IF + throw(6) + END
        body += lg(p) + ld32(8) + lg(2) + ADD32 + ls(e)
        body += lg(e) + c32(2) + SHL + ld32(self.setf) + IF + throw(3) + END
        body += c32(CELL_COUNT) + ld32() + c32(self.input_size) + GE_U + IF + throw(2) + END
        body += lg(e) + c32(2) + SHL + c32(1) + st32(self.setf)
        body += c32(CELL_COUNT) + c32(CELL_COUNT) + ld32() + c32(1) + ADD32 + st32()
        for j in range(8):
            body += lg(e) + c32(5) + SHL + c32(4 * j) + ld32() + st32(self.wires + 32 + 4 * j)
        if self.mode is not None:
            k = [n for n, _ in self.signals].index(self.mode)
            body += lg(s) + c32(k) + EQ + IF + c32(CELL_MODE) + c32(SHARED) + ld32() + st32() + END
        body += c32(CELL_COUNT) + ld32() + c32(self.input_size) + EQ + IF + call(COMPUTE) + END
        return A.Func([A.I32] * 3, [], body, locals_=[A.I32] * 3, export='setInputSignal')

    def _wsize(self):
        if self.claimed_size is not None:
            return c32(self.claimed_size)
        body = c32(self.n_wit)
        if self.protocol_fault:
            body += c32(CELL_INIT) + ld32() + ADD32
        if self.mode is not None:
            body += c32(CELL_MODE) + ld32() + c32(8) + EQ + ADD32
        return body

    def _module(self):
        init = c32(CELL_INIT) + c32(1) + st32() + (call(COMPUTE) if self.input_size == 0 else b'')
        prime = b''.join(c32(4 * j) + c32(RADDR + 4 * j) + ld32() + st32() for j in range(8))
        getw = b''.join(c32(4 * j) + lg(0) + c32(5) + SHL + ld32(self.wires + 4 * j) + st32() for j in range(8))
        fs = [self._add(), self._compute(),                                      # 4, 5 (ADD, COMPUTE)
              A.Func([], [A.I32], c32(2), export='getVersion'),
              A.Func([], [A.I32], c32(8), export='getFieldNumLen32'),
              A.Func([], [], prime, export='getRawPrime'),
              A.Func([], [A.I32], self._wsize(), export='getWitnessSize'),
              A.Func([], [A.I32], c32(self.input_size), export='getInputSize'),
              A.Func([A.I32], [], init, export='init'),
              A.Func([A.I32, A.I32], [], lg(0) + c32(2) + SHL + lg(1) + st32(), export='writeSharedRWMemory'),
              A.Func([A.I32], [A.I32], lg(0) + c32(2) + SHL + ld32(), export='readSharedRWMemory'),
              self._set_input(),
              A.Func([A.I32], [], getw, export='getWitness')]
        table = b''
        for n, sz in self.signals:
            h = fnv1a64(n)
            table += struct.pack('<IIII', h >> 32, h & M32, self.first[n], sz)
        imports = [('runtime', 'exceptionHandler', [A.I32], []), ('runtime', 'printErrorMessage', [], []),
                   ('runtime', 'writeBufferMessage', [], []), ('runtime', 'showSharedRWMemory', [], [])]
        return A.module(fs, memory=(self.pages, None), imports=imports,
                        data=[(RADDR, R_MOD.to_bytes(32, 'little')), (TAB, table)])
