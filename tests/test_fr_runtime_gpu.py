"""circom 2's field runtime on the device interpreter (csrc/wasm.cu): every case of tests/fr_runtime.py, one lane per
(case, window word), must end with the model's status and return the model's word, and the words must decode to the
big-integer result.  The cases are shuffled, so each warp mixes operand forms and branches."""
import numpy as np
import pytest

import fr_runtime as F
import wasm_model as M
from circom_compat_b200 import WasmModule

pytestmark = pytest.mark.gpu

NAMES = [s.name for s in F.build_specs()]


@pytest.fixture(scope='module')
def suite():
    return F.Suite(F.golden('circuit2.wasm'))


@pytest.fixture(scope='module')
def dev(ctx, suite):
    d = WasmModule(suite.data, ctx)
    d.set_limits(max_pages=F.PAGES)
    yield d
    d.close()


def _spec(suite, name):
    return next(s for s in suite.specs if s.name == name)


def _run(dev, sp, cases=None, fuel=None):
    """(results, statuses), each cases x len(sp.words), under the fuel the model gets"""
    cases = sp.cases if cases is None else cases
    rows = [(c.xp, c.yp, w) for c in cases for w in sp.words]
    dev.set_limits(fuel=sp.fuel if fuel is None else fuel)
    res, st = dev.run('t_' + sp.name, rows)
    return res.reshape(len(cases), len(sp.words)), st.reshape(len(cases), len(sp.words))


@pytest.mark.parametrize('name', NAMES)
def test_device_runtime_matches_model_and_big_integers(suite, dev, name):
    sp = _spec(suite, name)
    res, st = _run(dev, sp)
    for k, c in enumerate(sp.cases):
        ms, win = suite.run_model(sp, c)
        where = f"{name}(x={c.x:#x} {c.xf}, y={c.y if c.y is None else hex(c.y)} {c.yf})"
        assert (st[k] == ms).all(), (where, [int(s) for s in st[k]], ms)
        if ms != M.OK:
            continue
        want = F.words(win)
        got = [int(v) for v in res[k]]
        assert got == [want[w] for w in sp.words], (where, [hex(v) for v in got], [hex(want[w]) for w in sp.words])
        dwin = bytearray(F.WINDOW)                      # the device's words back in place: decode them on their own
        for w, v in zip(sp.words, got):
            dwin[8 * w:8 * w + 8] = v.to_bytes(8, 'little')
        sp.check(c, dwin, int(st[k][0]))


def test_chunked_runs_give_the_same_words(suite, dev):
    """a budget that fits a few warps splits the batch into many chunks; every word and status stays the same"""
    sp = _spec(suite, 'Fr_shr')
    whole = _run(dev, sp)
    lim = dev.limits
    per_lane = lim.max_pages * 65536 + lim.stack_slots * 8 + lim.max_depth * 8 + 3 * 8 + 8 + 4
    dev.set_limits(budget_bytes=per_lane * 100)         # 96 lanes a chunk
    try:
        parts = _run(dev, sp)
    finally:
        dev.set_limits(budget_bytes=0)
    assert whole[0].size > 20 * 96
    assert np.array_equal(whole[0], parts[0]) and np.array_equal(whole[1], parts[1])


def test_nonsquare_sqrt_runs_out_of_fuel_on_both(suite, dev):
    sp = _spec(suite, 'Fr_F1m_sqrt')
    cases = suite.nonsquare
    _, st = _run(dev, sp, cases, fuel=F.NONSQUARE_FUEL)
    for k, c in enumerate(cases):
        ms = suite.run_model(sp, c, fuel=F.NONSQUARE_FUEL)[0]
        assert (st[k] == ms).all(), (k, ms, st[k])
    assert (st == M.FUEL).all()
