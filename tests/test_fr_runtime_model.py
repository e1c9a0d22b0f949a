"""circom 2's field runtime on the plain-Python model (tests/wasm_model.py), one function at a time, against big-integer
arithmetic mod r at the edge operands of tests/fr_runtime.py.  The device test (test_fr_runtime_gpu.py) holds
csrc/wasm.cu to the same cases word for word; this file makes sure the cases themselves are right and keep reaching the
runtime's branches."""
import pytest

import fr_runtime as F
import wasm_model as M

NAMES = [s.name for s in F.build_specs()]

# instructions of each runtime function the case set executes on the model (the pcs of Module.body), as a floor: a
# change to the cases that lowers one of these drops a branch.  Fr_F1m_load, Fr_F1m_timesScalar, Fr_copyn and the *Old
# functions are left out: none of the tested functions calls them.
COVERAGE = {
    'int_copy': 17, 'int_zero': 13, 'int_isZero': 22, 'int_one': 13, 'int_eq': 30, 'int_gt': 54, 'int_gte': 54,
    'int_add': 105, 'int_sub': 121, 'int_mul': 1037, 'int_square': 1153, 'int__mul1': 93, 'int__add1': 37,
    'int_div': 142, 'int_inverseMod': 113, 'F1m_add': 17, 'F1m_sub': 12, 'F1m_neg': 5, 'F1m_mReduct': 1081,
    'F1m_mul': 2005, 'F1m_square': 2121, 'F1m_toMontgomery': 5, 'F1m_fromMontgomery': 9, 'F1m_isNegative': 8,
    'F1m_inverse': 11, 'F1m_one': 4, 'F1m_exp': 151, 'F1m_sqrt': 94, 'F1m_isSquare': 14, 'copy': 21, 'isTrue': 16,
    'rawCopyS2L': 38, 'toMontgomery': 41, 'toNormal': 23, 'toLongNormal': 33, 'isNegative': 18, 'neg': 61,
    'getLsb32': 13, 'toInt': 14, 'add': 207, 'sub': 207, 'eqR': 154, 'gtR': 67, 'eq': 13, 'neq': 13, 'gt': 22,
    'geq': 22, 'lt': 22, 'leq': 22, 'mul': 211, 'idiv': 51, 'mod': 51, 'inv': 46, 'div': 8, 'pow': 35,
    'fixedShl': 10, 'fixedShr': 10, 'rawgetchunk': 13, 'rawshll': 54, 'rawshrl': 52, 'adjustBinResult': 23,
    'rawshl': 124, 'rawshr': 70, 'shl': 41, 'shr': 41, 'rawbandl': 29, 'band': 215, 'rawborl': 29, 'bor': 215,
    'rawbxorl': 29, 'bxor': 215, 'rawbnotl': 25, 'bnot': 31, 'land': 15, 'lor': 15, 'lnot': 12,
}


@pytest.fixture(scope='module')
def runs():
    """every case once on the model, with the executed-pc trace on: (suite, {name: [(status, window)]}, trace)"""
    s = F.Suite(F.golden('circuit2.wasm'))
    trace = {}
    out = {sp.name: [s.run_model(sp, c, trace=trace) for c in sp.cases] for sp in s.specs}
    return s, out, trace


@pytest.mark.parametrize('name', NAMES)
def test_model_matches_big_integers(runs, name):
    s, out, _ = runs
    sp = next(x for x in s.specs if x.name == name)
    assert sp.cases
    for c, (st, win) in zip(sp.cases, out[name]):
        try:
            sp.check(c, win, st)
        except AssertionError as e:
            raise AssertionError(f"{name}(x={c.x:#x} {c.xf}, y={c.y if c.y is None else hex(c.y)} {c.yf}): {e}")


def test_every_element_operator_sees_every_form_pair():
    for sp in F.build_specs():
        if sp.name in F.ELEMENT_BINARY:
            assert {(c.xf, c.yf) for c in sp.cases} == {(a, b) for a in 'slm' for b in 'slm'}, sp.name
        elif sp.cases[0].xf:                                     # the unary element functions
            assert {c.xf for c in sp.cases} == set('slm'), sp.name


def test_edge_values_reach_every_element_operator():
    """each edge value that fits a form is an x operand in that form, and a y operand where y is an element"""
    for sp in F.build_specs():
        if sp.name not in F.ELEMENT_BINARY and sp.name not in F.ELEMENT_UNARY:
            continue
        for f in 'slm':
            xs = {c.x for c in sp.cases if c.xf == f}
            want = {v for v in F.E if F.representable(v, f)}
            if sp.name not in ('Fr_div', 'Fr_pow', 'Fr_inv'):      # the costly ones take a sample
                assert want <= xs, (sp.name, f, want - xs)


def test_runtime_bodies_are_the_same_in_both_golden_modules():
    """testing circuit2's runtime covers mycircuit's: same indices, byte-identical bodies"""
    a, b = F.golden('circuit2.wasm'), F.golden('mycircuit.wasm')
    na, nb = F.function_names(a), F.function_names(b)
    rt = sorted(n for n in na if n.startswith('Fr_'))
    assert len(rt) >= 80 and rt == sorted(n for n in nb if n.startswith('Fr_'))
    for n in rt:
        assert na[n] == nb[n] and F.function_body(a, n) == F.function_body(b, n), n


def test_patch_leaves_the_module_alone():
    """the patched module keeps every original function body, data segment, export and the name section's indices"""
    data = F.golden('circuit2.wasm')
    s = F.Suite(data)
    m0, m1 = M.Module(data), s.module
    assert m1.mem == (F.PAGES, None) and m0.mem == (F.PAGES - 1, None)
    for k, (_, st, en) in enumerate(m0.codes):
        _, st1, en1 = m1.codes[k]
        assert data[st:en] == s.data[st1:en1], k
    assert m1.datas[:-1] == m0.datas and m1.datas[-1] == (('i32', F.TABLE), s.table)
    assert all(m1.exports[k] == v for k, v in m0.exports.items())
    assert F.function_names(s.data) == F.function_names(data)
    assert {'t_' + sp.name for sp in s.specs} <= set(m1.exports)


def test_coverage_floor(runs):
    s, _, trace = runs
    m = s.module
    names = F.function_names(s.data)
    got = {}
    for n, i in names.items():
        if n.startswith('Fr_') and n[3:] in COVERAGE:
            got[n[3:]] = len(trace.get(i - len(m.imports), ()))
    low = {n: (got[n], f) for n, f in COVERAGE.items() if got[n] < f}
    assert not low, low


def test_nonsquare_sqrt_runs_out_of_fuel():
    """Fr_F1m_sqrt of a non-square never ends (the root search finds no root): under a small fuel it stops with FUEL"""
    s = F.Suite(F.golden('circuit2.wasm'))
    sp = next(x for x in s.specs if x.name == 'Fr_F1m_sqrt')
    for c in s.nonsquare:
        assert s.run_model(sp, c, fuel=F.NONSQUARE_FUEL)[0] == M.FUEL
