"""circom 2's field runtime (the ~80 Fr_* functions every circom 2 module carries) called one function at a time, on the
model and on the device, at the operands where its branches split.

A circom 2 module names every function in its `name` custom section; the runtime's functions are Fr_int_* (raw 256-bit
integers), Fr_F1m_* (Montgomery arithmetic, R = 2^256) and Fr_* (field elements).  An element is 40 bytes: an i32
short value, an i32 type word (bit 31: long, bit 30: Montgomery), then 8 little-endian limbs.

patch(data, specs) returns the module with one more memory page and, in it, an operand table, a fixed result window
and one exported wrapper per tested function:

    t_<name>(x_ptr, y_ptr, w) -> i64
        copies the 64-byte table entries at x_ptr and y_ptr to X and Y, calls <name> with its arguments drawn from
        R (the result area), R + 32, X, Y and constants, stores an i32 result at RET and returns i64 word w of the
        window.  The runtime converts operands in place, so the copies keep the table intact and show what the
        function did to its operands.

The rest of the module is unchanged, so the function indices stay the ones the name section gives.
"""
from __future__ import annotations

import os
import random
import struct

import wasm_asm as A
import wasm_model as M

R = M.R_MOD
PAGE = M.PAGE
M32 = M.M32
RINV = pow(1 << 256, -1, R)
MASK254 = (1 << 254) - 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

PAGES = 12                       # the golden modules declare 11 initial pages and no maximum
BASE = (PAGES - 1) * PAGE        # the window: R (64 B), X (64 B), Y (64 B), RET (8 B)
RES, XC, YC, RET = BASE, BASE + 64, BASE + 128, BASE + 192
WINDOW = 200
TABLE = BASE + 256
ENTRY = 64
# the runtime's own scratch in low memory: the constants and the temporaries below 2032 + 4096 it works in
SCRATCH_END = 2032 + 4096
# the fuel (instructions) a call may use: about twice the most a case takes on the model, so that an interpreter bug
# that sends the runtime into an endless loop ends that lane with FUEL in seconds
FUEL = 20000
STEPS = {'Fr_div': 10 ** 6, 'Fr_pow': 2 * 10 ** 6, 'Fr_idiv': 2 * 10 ** 5, 'Fr_mod': 2 * 10 ** 5, 'Fr_inv': 10 ** 6,
         'Fr_int_div': 2 * 10 ** 5, 'Fr_int_inverseMod': 10 ** 6, 'Fr_F1m_inverse': 10 ** 6, 'Fr_F1m_isSquare': 2 * 10 ** 6,
         'Fr_F1m_sqrt': 5 * 10 ** 6, 'Fr_F1m_exp': 2 * 10 ** 6}
NONSQUARE_FUEL = 20000    # Fr_F1m_sqrt of a non-square never returns: it runs until the fuel is gone


def golden(name):
    return open(os.path.join(GOLDEN, name), 'rb').read()


# -------------------------------------------------------------------------------------------------------- the module
def _sections(data):
    r = M._Reader(data, 8)
    out = []
    while r.p < len(data):
        sid, size = r.byte(), r.uleb()
        out.append((sid, bytes(data[r.p:r.p + size])))
        r.p += size
    return out


def function_names(data) -> dict:
    """{name: function index} from the `name` custom section (subsection 1, the function names)"""
    names = {}
    for sid, body in _sections(data):
        if sid != 0:
            continue
        s = M._Reader(body)
        if s.name() != 'name':
            continue
        while s.p < s.end:
            sub, size = s.byte(), s.uleb()
            end = s.p + size
            if sub == 1:
                for _ in range(s.uleb()):
                    i = s.uleb()
                    names[s.name()] = i
            s.p = end
    return names


def function_body(data, name) -> bytes:
    """the code-section bytes (locals and instructions) of a named function"""
    m = M.Module(data)
    _, start, end = m.codes[function_names(data)[name] - len(m.imports)]
    return bytes(data[start:end])


def _append_vec(body: bytes, items) -> bytes:
    r = M._Reader(body)
    n = r.uleb()
    return A.uleb(n + len(items)) + body[r.p:] + b''.join(items)


def _wrapper(f, pattern, ret):
    """the body of t_<name>: copy the operands, call f, store its i32 result, return word w of the window"""
    b = b''
    for dst, src in ((XC, 0), (YC, 1)):
        for j in range(0, ENTRY, 8):
            b += A.i32c(dst + j) + A.lget(src) + A.memarg(0x29, j, 3) + A.memarg(0x37, 0, 3)
    if ret:
        b += A.i32c(RET)
    for p in pattern:
        b += A.i32c({'r': RES, 'r2': RES + 32, 'x': XC, 'y': YC}[p] if isinstance(p, str) else p)
    b += b'\x10' + A.uleb(f)
    if ret:
        b += A.memarg(0x36, 0, 2)
    b += A.i32c(BASE) + A.lget(2) + A.i32c(3) + b'\x74\x6a' + A.memarg(0x29, 0, 3)
    return b


def patch(data: bytes, specs, table: bytes) -> bytes:
    """the module with PAGES initial pages, `table` at TABLE and an export t_<name> per spec"""
    idx = function_names(data)
    m = M.Module(data)
    assert m.mem == (PAGES - 1, None), m.mem
    assert TABLE + len(table) <= PAGES * PAGE
    tw = len(m.types)
    fns, exps, codes = [], [], []
    for k, s in enumerate(specs):
        f = idx[s.name]
        ps, rs = m.ftype(f)
        assert len(ps) == len(s.pattern) and rs == ((A.I32,) if s.ret else ()), (s.name, ps, rs)
        fns.append(A.uleb(tw))
        exps.append(A.name('t_' + s.name) + b'\x00' + A.uleb(len(m.imports) + len(m.codes) + k))
        body = b'\x00' + _wrapper(f, s.pattern, s.ret) + b'\x0b'
        codes.append(A.uleb(len(body)) + body)
    out = bytearray(data[:8])
    for sid, body in _sections(data):
        if sid == 1:
            body = _append_vec(body, [b'\x60' + A.vec([bytes([A.I32])] * 3) + A.vec([bytes([A.I64])])])
        elif sid == 3:
            body = _append_vec(body, fns)
        elif sid == 5:
            body = A.vec([b'\x00' + A.uleb(PAGES)])
        elif sid == 7:
            body = _append_vec(body, exps)
        elif sid == 10:
            body = _append_vec(body, codes)
        elif sid == 11:
            body = _append_vec(body, [b'\x00' + A.i32c(TABLE) + b'\x0b' + A.uleb(len(table)) + table])
        out += A.section(sid, body)
    return bytes(out)


# -------------------------------------------------------------------------------------------------------- operands
def representable(v, form):
    """short elements hold the i32 range of the signed value: [0, 2^31) and [r - 2^31, r)"""
    return form != 's' or v < 1 << 31 or R - v <= 1 << 31


def element(v, form) -> bytes:
    if form == 's':
        s = v if v < 1 << 31 else v - R
        return struct.pack('<iI', s, 0) + bytes(32)
    if form == 'l':
        return struct.pack('<iI', 0, 0x80000000) + v.to_bytes(32, 'little')
    return struct.pack('<iI', 0, 0xC0000000) + (v * (1 << 256) % R).to_bytes(32, 'little')


def decode(b):
    """(value mod r, form) of a 40-byte element; a long limb vector >= r is reported as form 'bad'"""
    s, t = struct.unpack('<iI', bytes(b[:8]))
    v = int.from_bytes(bytes(b[8:40]), 'little')
    if not t >> 31:
        return s % R, 's'
    if v >= R:
        return v, 'bad'
    return (v * RINV % R, 'm') if t >> 30 & 1 else (v, 'l')


def sval(v):
    """the signed value circom compares: v - r above r // 2"""
    return v - R if v > R // 2 else v


E = [0, 1, 2, 3, 253, 254, 255, 256, (1 << 31) - 1, (1 << 31) + 1, (1 << 32) - 1, (1 << 32) + 1, (1 << 64) - 1,
     (1 << 64) + 1, R // 2 - 1, R // 2, R // 2 + 1, R - 1, R - 2, R - 253, R - 254, R - 255, R - (1 << 31),
     R - (1 << 31) - 1, 1 << 253, MASK254 % R]
_LIMBS = [(1 << (64 * k)) + d for k in (1, 2, 3) for d in (-1, 0, 1)] + [(1 << 256) - (1 << 64), (1 << 192) - 1]
RAW = sorted(set(E + _LIMBS + [(1 << 256) - 1, (1 << 256) - 2, 1 << 255, R, R + 1, 2 * R, 2 * R - 1]))
SHIFTS = [0, 1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 253, 254, 255, 256, 1000, R - 1, R - 2, R - 31,
          R - 64, R - 253, R - 254, R - 255, R - 256, R // 2, R // 2 + 1, R // 2 - 1]


def _random_values(rng):
    return [rng.randrange(R) for _ in range(6)] + [rng.randrange(1 << 31) for _ in range(2)] + \
        [R - rng.randrange(1, 1 << 31) for _ in range(2)] + [rng.randrange(1 << 64) for _ in range(2)]


# -------------------------------------------------------------------------------------------------------- semantics
def _idiv(a, b):
    if b == 0:
        raise ZeroDivisionError
    return a // b


def _shr(a, k):
    return (a >> k if k < 254 else 0) if k <= R // 2 else _shl(a, R - k)


def _shl(a, k):
    return (((a << k) & MASK254) % R if k < 254 else 0) if k <= R // 2 else _shr(a, R - k)


def _inv(a):
    return pow(a, -1, R) if a else 0


ELEMENT_BINARY = {
    'Fr_add': lambda a, b: (a + b) % R, 'Fr_sub': lambda a, b: (a - b) % R, 'Fr_mul': lambda a, b: a * b % R,
    'Fr_div': lambda a, b: a * _inv(b) % R, 'Fr_pow': lambda a, b: pow(a, b, R),
    'Fr_idiv': _idiv, 'Fr_mod': lambda a, b: a - _idiv(a, b) * b,
    'Fr_eq': lambda a, b: int(a == b), 'Fr_neq': lambda a, b: int(a != b),
    'Fr_lt': lambda a, b: int(sval(a) < sval(b)), 'Fr_gt': lambda a, b: int(sval(a) > sval(b)),
    'Fr_leq': lambda a, b: int(sval(a) <= sval(b)), 'Fr_geq': lambda a, b: int(sval(a) >= sval(b)),
    'Fr_land': lambda a, b: int(bool(a) and bool(b)), 'Fr_lor': lambda a, b: int(bool(a) or bool(b)),
    'Fr_band': lambda a, b: (a & b) % R, 'Fr_bor': lambda a, b: (a | b) % R, 'Fr_bxor': lambda a, b: (a ^ b) % R,
    'Fr_shl': _shl, 'Fr_shr': _shr,
}
ELEMENT_UNARY = {
    'Fr_neg': lambda a: -a % R, 'Fr_inv': _inv, 'Fr_copy': lambda a: a, 'Fr_lnot': lambda a: int(a == 0),
    'Fr_bnot': lambda a: (~a & MASK254) % R,
}


class Spec:
    """one tested function: its argument pattern, whether it returns an i32, the window words the device reads and
    check(case, window) -> None, which asserts the big-int semantics"""

    def __init__(self, name, pattern, ret, words, check, cases=None):
        self.name, self.pattern, self.ret, self.words, self.check = name, tuple(pattern), ret, list(words), check
        self.cases = cases or []
        self.fuel = STEPS.get(name, FUEL)


W_RES = lambda n: list(range(n))                 # noqa: E731  the first n words of R
W_X = list(range(8, 13))                         # the element copy at X
W_Y = list(range(16, 21))
W_RET = [24]


class Case:
    def __init__(self, x, y, xb, yb, xf='', yf=''):
        self.x, self.y, self.xb, self.yb, self.xf, self.yf = x, y, xb, yb, xf, yf


def _res_int(win, off=0, n=32):
    return int.from_bytes(bytes(win[off:off + n]), 'little')


def _ret(win):
    return struct.unpack('<I', bytes(win[192:196]))[0]


def _check_element(fn):
    def check(c, win, status):
        try:
            want = fn(c.x, c.y) if c.yf else fn(c.x)
        except ZeroDivisionError:
            assert status == M.DIV_ZERO, status
            return
        assert status == M.OK, status
        v, form = decode(win[0:40])
        assert form != 'bad' and v == want, (v, form, want)
    return check


def _near(rng):
    """pairs that agree in their high limbs and differ in one lower limb, and equal pairs: the limb-by-limb compare
    loops run to their last limb only on these"""
    v = rng.randrange(1 << 192, R - (1 << 193))
    d = [0, 1, 1 << 32, 1 << 64, 1 << 128, 1 << 160, 1 << 192]
    return [(v, v + x) for x in d] + [(v + x, v) for x in d[1:]] + [(R - 1, R - 1), (R // 2, R // 2 + 1)]


def _form_pairs(rng, values, pairs_per_form=None, forms='slm', second=None):
    """every form pair; in each, every representable value appears as x and as y at least once (or a random sample of
    pairs_per_form pairs)"""
    out = []
    near = _near(rng) if second is None else []
    second = second if second is not None else values
    for fa in forms:
        for fb in forms:
            va = [v for v in values if representable(v, fa)]
            vb = [v for v in second if representable(v, fb)]
            ps = [(a, rng.choice(vb)) for a in va] + [(rng.choice(va), b) for b in vb]
            ps += [(a, b) for a, b in near if representable(a, fa) and representable(b, fb)]
            if pairs_per_form is not None:
                ps = rng.sample(ps, min(pairs_per_form, len(ps)))
            out += [Case(a, b, element(a, fa), element(b, fb), fa, fb) for a, b in ps]
    return out


def _unary_forms(rng, values, per_form=None):
    out = []
    for fa in 'slm':
        va = [v for v in values if representable(v, fa)]
        if per_form is not None:
            va = rng.sample(va, min(per_form, len(va)))
        out += [Case(a, None, element(a, fa), bytes(40), fa) for a in va]
    return out


def _raw(v, n=32):
    return v.to_bytes(n, 'little')


def _raw_pairs(rng, xs, ys=None, n=None):
    ys = ys if ys is not None else xs
    ps = [(a, rng.choice(ys)) for a in xs] + [(rng.choice(xs), b) for b in ys] + [(b, b) for b in ys[:8]]
    if n is not None:
        ps = rng.sample(ps, min(n, len(ps)))
    return [Case(a, b, _raw(a), _raw(b)) for a, b in ps]


def build_specs(seed=2024):
    rng = random.Random(seed)
    ev = E + _random_values(rng)
    specs = []
    small = {'Fr_div': 4, 'Fr_pow': 2}                      # an inversion or a 254-bit exponent: 0.3 to 0.8 M steps
    for name, fn in ELEMENT_BINARY.items():
        ys = SHIFTS if name in ('Fr_shl', 'Fr_shr') else None
        if name == 'Fr_pow':
            ys = [0, 1, 2, 3, R - 1, R - 2, (1 << 64) - 1, rng.randrange(R)]
        cases = _form_pairs(rng, ev, small.get(name), second=ys)
        specs.append(Spec(name, ('r', 'x', 'y'), False, W_RES(5) + W_X + W_Y, _check_element(fn), cases))
    for name, fn in ELEMENT_UNARY.items():
        cases = _unary_forms(rng, ev, 4 if name == 'Fr_inv' else None)
        specs.append(Spec(name, ('r', 'x'), False, W_RES(5) + W_X, _check_element(fn), cases))
    # i32 results of one element
    # toInt is the low word of the signed value; getLsb32 that of a short's value but of the canonical limbs of a long
    preds = {'Fr_isTrue': lambda a, f: int(a != 0), 'Fr_isNegative': lambda a, f: int(a > R // 2),
             'Fr_toInt': lambda a, f: sval(a) & M32, 'Fr_getLsb32': lambda a, f: (sval(a) if f == 's' else a) & M32}
    for name, fn in preds.items():
        def chk(c, win, st, fn=fn):
            assert st == M.OK and _ret(win) == fn(c.x, c.xf), (st, _ret(win), fn(c.x, c.xf))
        specs.append(Spec(name, ('x',), True, W_X + W_RET, chk, _unary_forms(rng, ev)))
    # in-place conversions: the value stays, the form changes
    conv = {'Fr_toMontgomery': ('m', 's'), 'Fr_toNormal': ('l', 's'), 'Fr_toLongNormal': ('l',)}
    for name, forms in conv.items():
        def chk(c, win, st, forms=forms, name=name):
            v, form = decode(win[64:104])
            assert st == M.OK and v == c.x and (form in forms if c.xf != 's' or name == 'Fr_toLongNormal' else True), \
                (st, v, form)
            if name == 'Fr_toLongNormal':
                assert form == 'l'
            elif c.xf != 's':
                assert form == forms[0], (name, c.xf, form)
        specs.append(Spec(name, ('x',), False, W_X, chk, _unary_forms(rng, ev)))
    specs += _raw_specs(rng)
    specs += _f1m_specs(rng, ev)                              # F1m operands are residues < r
    return specs


def _raw_specs(rng):
    specs = []
    T = 1 << 256

    def chk_add(c, win, st):
        s = c.x + c.y
        assert st == M.OK and _res_int(win) == s % T and _ret(win) == s >> 256
    specs.append(Spec('Fr_int_add', ('x', 'y', 'r'), True, W_RES(4) + W_RET, chk_add, _raw_pairs(rng, RAW)))

    def chk_sub(c, win, st):
        assert st == M.OK and _res_int(win) == (c.x - c.y) % T and _ret(win) == (M32 if c.x < c.y else 0)
    specs.append(Spec('Fr_int_sub', ('x', 'y', 'r'), True, W_RES(4) + W_RET, chk_sub, _raw_pairs(rng, RAW)))

    def chk_mul(c, win, st):
        assert st == M.OK and _res_int(win, 0, 64) == c.x * c.y
    specs.append(Spec('Fr_int_mul', ('x', 'y', 'r'), False, W_RES(8), chk_mul, _raw_pairs(rng, RAW)))

    def chk_sq(c, win, st):
        assert st == M.OK and _res_int(win, 0, 64) == c.x * c.x
    specs.append(Spec('Fr_int_square', ('x', 'r'), False, W_RES(8), chk_sq, _raw_pairs(rng, RAW)))
    for name, fn in (('Fr_int_gt', lambda a, b: a > b), ('Fr_int_gte', lambda a, b: a >= b),
                     ('Fr_int_eq', lambda a, b: a == b)):
        def chk(c, win, st, fn=fn):
            assert st == M.OK and _ret(win) == int(fn(c.x, c.y))
        specs.append(Spec(name, ('x', 'y'), True, W_RET, chk, _raw_pairs(rng, RAW)))

    def chk_zero(c, win, st):
        assert st == M.OK and _ret(win) == int(c.x == 0)
    specs.append(Spec('Fr_int_isZero', ('x',), True, W_RET, chk_zero, _raw_pairs(rng, RAW)))

    def chk_div(c, win, st):
        assert st == M.OK and _res_int(win) == c.x // c.y and _res_int(win, 32) == c.x % c.y
    nz = [v for v in RAW if v]
    specs.append(Spec('Fr_int_div', ('x', 'y', 'r', 'r2'), False, W_RES(8), chk_div, _raw_pairs(rng, RAW, nz, 60)))

    def chk_invm(c, win, st):
        assert st == M.OK and _res_int(win) == pow(c.x, -1, c.y)
    inv_x = [v for v in E if v] + [rng.randrange(1, R) for _ in range(4)]
    cases = [Case(a, R, _raw(a), _raw(R)) for a in rng.sample(inv_x, 10)]
    specs.append(Spec('Fr_int_inverseMod', ('x', 'y', 'r'), False, W_RES(4), chk_invm, cases))
    return specs


def _f1m_specs(rng, vals):
    T = 1 << 256
    specs = []
    bin_ = {'Fr_F1m_add': lambda a, b: (a + b) % R, 'Fr_F1m_sub': lambda a, b: (a - b) % R,
            'Fr_F1m_mul': lambda a, b: a * b * RINV % R}
    for name, fn in bin_.items():
        def chk(c, win, st, fn=fn):
            assert st == M.OK and _res_int(win) == fn(c.x, c.y)
        specs.append(Spec(name, ('x', 'y', 'r'), False, W_RES(4), chk, _raw_pairs(rng, vals)))
    un = {'Fr_F1m_neg': lambda a: -a % R, 'Fr_F1m_square': lambda a: a * a * RINV % R,
          'Fr_F1m_toMontgomery': lambda a: a * T % R, 'Fr_F1m_fromMontgomery': lambda a: a * RINV % R,
          'Fr_F1m_inverse': lambda a: pow(a, -1, R) * T * T % R if a else 0}
    for name, fn in un.items():
        def chk(c, win, st, fn=fn):
            assert st == M.OK and _res_int(win) == fn(c.x), (_res_int(win), fn(c.x))
        xs = rng.sample(vals, 8) if name == 'Fr_F1m_inverse' else vals
        specs.append(Spec(name, ('x', 'r'), False, W_RES(4), chk, [Case(a, None, _raw(a), bytes(32)) for a in xs]))

    def legendre(a):
        return pow(a * RINV % R, (R - 1) // 2, R)

    def chk_issq(c, win, st):
        assert st == M.OK and _ret(win) == int(legendre(c.x) != R - 1)
    specs.append(Spec('Fr_F1m_isSquare', ('x',), True, W_RET, chk_issq, [Case(a, None, _raw(a), bytes(32)) for a in vals]))
    squares = [0, T % R] + [a * a * RINV % R for a in (rng.randrange(R), rng.randrange(R), R - 1, 2, 5)]

    def chk_sqrt(c, win, st):
        s = _res_int(win)
        assert st == M.OK and s < R and s * s * RINV % R == c.x
    specs.append(Spec('Fr_F1m_sqrt', ('x', 'r'), False, W_RES(4), chk_sqrt, [Case(a, None, _raw(a), bytes(32)) for a in squares]))

    def chk_red(c, win, st):
        assert st == M.OK and _res_int(win) == c.x * RINV % R
    wide = [0, 1, R - 1, R * T - 1, (R - 1) * (R - 1), R, T, T - 1, R * (T - 1), rng.randrange(R * T)]
    specs.append(Spec('Fr_F1m_mReduct', ('x', 'r'), False, W_RES(4), chk_red,
                      [Case(a, None, _raw(a, 64), bytes(64)) for a in wide]))

    def chk_exp(c, win, st):
        b = c.x * RINV % R
        assert st == M.OK and _res_int(win) == pow(b, c.y, R) * T % R
    es = [0, 1, 2, 3, 255, 1 << 64, R - 1, rng.randrange(R)]
    cases = [Case(a, e, _raw(a), _raw(e)) for a, e in zip(rng.sample(vals, len(es)), es)]
    specs.append(Spec('Fr_F1m_exp', ('x', 'y', 32, 'r'), False, W_RES(4), chk_exp, cases))
    return specs


# -------------------------------------------------------------------------------------------------------- running
class Suite:
    """the specs, the operand table, the patched module and each case's (x_ptr, y_ptr); cases are shuffled so that a
    warp's lanes take different branches"""

    def __init__(self, data: bytes, seed=2024):
        self.specs = build_specs(seed)
        rng = random.Random(seed + 1)
        entries, at = [], {}

        def ptr(b):
            b = bytes(b).ljust(ENTRY, b'\0')
            if b not in at:
                at[b] = TABLE + ENTRY * len(entries)
                entries.append(b)
            return at[b]
        for s in self.specs:
            rng.shuffle(s.cases)
            for c in s.cases:
                c.xp, c.yp = ptr(c.xb), ptr(c.yb)
        # Fr_F1m_sqrt operands that are not squares (5 and r - 5 in Montgomery form; 5 is a non-residue mod r)
        self.nonsquare = [Case(v, None, _raw(v), bytes(32)) for v in (5 * (1 << 256) % R, (R - 5) * (1 << 256) % R)]
        for c in self.nonsquare:
            c.xp, c.yp = ptr(c.xb), ptr(c.yb)
        self.table = b''.join(entries)
        self.data = patch(data, self.specs, self.table)
        self.module = M.Module(self.data, protocol=False)
        self.pristine = bytes(M.Instance(self.module, max_pages=PAGES).mem)

    def run_model(self, spec, case, fuel=None, trace=None):
        """(status, window bytes) of one call on a fresh model instance under spec.fuel (or `fuel`); asserts it wrote
        only the window and the runtime's scratch"""
        inst = M.Instance(self.module, max_pages=PAGES, fuel=spec.fuel if fuel is None else fuel, trace=trace)
        try:
            inst.call('t_' + spec.name, case.xp, case.yp, 0)
            st = M.OK
        except M.Trap as t:
            st = t.status
        mem = inst.mem
        assert len(mem) == PAGES * PAGE, (spec.name, 'grew the memory')
        p = self.pristine
        assert mem[SCRATCH_END:BASE] == p[SCRATCH_END:BASE] and mem[BASE + WINDOW:] == p[BASE + WINDOW:], \
            (spec.name, 'wrote outside the window and the runtime scratch',
             next(i for i in range(SCRATCH_END, len(mem)) if mem[i] != p[i] and not BASE <= i < BASE + WINDOW))
        return st, bytes(mem[BASE:BASE + WINDOW])


def words(win):
    return [int.from_bytes(win[8 * w:8 * w + 8], 'little') for w in range(WINDOW // 8)]
