"""A small WebAssembly binary writer for hand-built test modules (no text format, no toolchain)."""
from __future__ import annotations

I32, I64, F32, F64 = 0x7f, 0x7e, 0x7d, 0x7c


def uleb(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def sleb(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        done = (v == 0 and not b & 0x40) or (v == -1 and b & 0x40)
        out.append(b | (0 if done else 0x80))
        if done:
            return bytes(out)


def name(s: str) -> bytes:
    return uleb(len(s)) + s.encode()


def vec(items) -> bytes:
    items = list(items)
    return uleb(len(items)) + b''.join(items)


def section(sid: int, body: bytes) -> bytes:
    return bytes([sid]) + uleb(len(body)) + body


def i32c(v: int) -> bytes:
    return b'\x41' + sleb(v - (1 << 32) if v >= 1 << 31 else v)


def i64c(v: int) -> bytes:
    return b'\x42' + sleb(v - (1 << 64) if v >= 1 << 63 else v)


def lget(i: int) -> bytes:
    return b'\x20' + uleb(i)


def memarg(op: int, offset: int = 0, align: int = 0) -> bytes:
    return bytes([op]) + uleb(align) + uleb(offset)


class Func:
    def __init__(self, params, results, body: bytes, locals_=(), export: str = None):
        self.params, self.results, self.body, self.locals, self.export = tuple(params), tuple(results), body, list(locals_), export


def module(funcs, memory=None, data=(), imports=(), globals_=(), table=None, elems=(), raw_sections=()) -> bytes:
    """funcs: [Func]; memory: (min, max or None); data: [(offset, bytes)]; imports: [(module, name, params, results)];
    globals_: [(type, mutable, init expr bytes)]; table: size; elems: [(offset, [function indices])]"""
    types = []

    def tidx(ps, rs):
        t = (tuple(ps), tuple(rs))
        if t not in types:
            types.append(t)
        return types.index(t)
    imp = [name(m) + name(n) + b'\x00' + uleb(tidx(ps, rs)) for m, n, ps, rs in imports]
    fidx = [uleb(tidx(f.params, f.results)) for f in funcs]
    out = b'\0asm\x01\0\0\0'
    out += section(1, vec(b'\x60' + vec(bytes([p]) for p in ps) + vec(bytes([r]) for r in rs) for ps, rs in types))
    if imp:
        out += section(2, vec(imp))
    out += section(3, vec(fidx))
    if table is not None:
        out += section(4, vec([b'\x70\x00' + uleb(table)]))
    if memory is not None:
        lo, hi = memory
        out += section(5, vec([(b'\x00' + uleb(lo)) if hi is None else (b'\x01' + uleb(lo) + uleb(hi))]))
    if globals_:
        out += section(6, vec(bytes([t, m]) + init + b'\x0b' for t, m, init in globals_))
    nimp = len(imports)
    exps = [name(f.export) + b'\x00' + uleb(nimp + k) for k, f in enumerate(funcs) if f.export]
    out += section(7, vec(exps))
    if elems:
        out += section(9, vec(b'\x00' + i32c(off) + b'\x0b' + vec(uleb(x) for x in fs) for off, fs in elems))
    bodies = []
    for f in funcs:
        groups = b''.join(uleb(1) + bytes([t]) for t in f.locals)
        b = uleb(len(f.locals)) + groups + f.body + b'\x0b'
        bodies.append(uleb(len(b)) + b)
    out += section(10, vec(bodies))
    if data:
        out += section(11, vec(b'\x00' + i32c(off) + b'\x0b' + uleb(len(d)) + d for off, d in data))
    for sid, body in raw_sections:
        out += section(sid, body)
    return out
