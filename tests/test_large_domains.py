"""The NTT from 2^23 to 2^27 and the setup, ceremony and key paths across their slice boundaries, at the sizes users run.

Every size here is chosen from a constant or a schedule rule in the CUDA sources; a change to one of them needs a matching
change here:

  constant / rule                                   value              reached by
  SETUP_SLICE     csrc/setup.cu:160 (setup_points)  2^20 points        setup with 2^20 + 37 variables (H of 2^21 rows)
  KEY_SLICE       csrc/verify.cu:620 (points_slices) 2^20 points       (de)serialization of 2^20 + 5 points
  PREP_PINNED     csrc/setup.cu:834 (to_host)       64 MiB             prepare at power 20: tau_g1 block 21 = 128 MiB,
                                                                       tau_g2 block 20 = 128 MiB, tau_g1 block 20 = 64 MiB
  POWERS_SLICE    csrc/msm.cuh:75 (b2g_setup_check) 2^22 points        key check with 2^22 + 37 variables
  NTT passes      csrc/ntt.cu:403-423               block pass of 10 index bits, then strided passes of at most 7 bits
                  (ntt_domain_create)               (2-D tiles from 2^21), at most three:
                                                      2^23: 10 | 6, 7          2^24: 10 | 7, 7
                                                      2^25: 10 | 5, 5, 5       2^26: 10 | 5, 5, 6      2^27: 10 | 5, 6, 6
                                                      2^23, B2G_NTT_MAXK=5: 10 | 4, 4, 5 (the cap of three passes)
                                                      2^23, B2G_NTT_RADIX2=1: the one-stage-per-barrier kernel, 10 | 6, 7

References are independent of the path under test: oracle/cref.c, big-int closed forms, synth.setup_scalars, the
fixed-base entry points (b2g_fixed_base_*, which do not go through setup_points) and single-slice calls of the same entry
point.  A vector of 2^27 field elements is 4 GiB; no test holds more than three such host arrays at once."""
import ctypes as C
import random

import numpy as np
import pytest

import ark_key_model as M
from batch_model import twist_point_outside_g2
from compressed_model import P, g1_no_root_x, g2_bytes, g2_no_root_x
from circom_compat_b200 import (CircomReduction, Groth16, LibsnarkReduction, Powers, ProvingKey, read_ptau, release,
                                synth)
from circom_compat_b200 import _native as N
from circom_compat_b200 import verifier as V
from circom_compat_b200.ptau import ARRAYS, LAGRANGE
from circom_compat_b200.zkey import ConstraintMatrices, csr_from_coo
from oracle import cref as c

R = c.R_MOD
SETUP_SLICE = 1 << 20
KEY_SLICE = 1 << 20
PREP_PINNED = 64 << 20
POWERS_SLICE = 1 << 22
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


# ---------------------------------------------------------------------------------------------------------------- helpers
def _schedule(log_n, radix2=False, maxk=None):
    """(block-pass bits, [(first bit, bits) of each strided pass]) as ntt_domain_create chooses them"""
    tl = min(log_n, 10)
    rem, passes, sb = log_n - tl, [], tl
    if rem > 0:
        k_max = maxk if maxk is not None else (7 if log_n > 20 and tl > 7 else tl)
        np_ = min(-(-rem // k_max), 3)
        for p in range(np_):
            k = rem // (np_ - p)
            passes.append((sb, k))
            sb += k
            rem -= k
    return tl, passes


def _checked_indices(log_n, seed, **kw):
    """every index within 2 of a multiple of a tile, row or pass boundary (first three multiples and the last), both ends,
    and 4096 random indices"""
    n = 1 << log_n
    tl, passes = _schedule(log_n, **kw)
    bits = {3, 5, tl} | {b for sb, k in passes for b in (sb, sb + k)}
    ks = set(range(3)) | set(range(n - 3, n))
    for b in bits:
        if b >= log_n:
            continue
        for m in (1, 2, 3, (n >> b) - 1):
            ks |= {m * (1 << b) + d for d in range(-2, 3)}
    ks |= set(np.random.default_rng(seed).integers(0, n, 4096).tolist())
    return np.array(sorted(k for k in ks if 0 <= k < n), dtype=np.int64)


def _mont(vals):
    return c.fr_to_mont(c.ints_to_limbs([v % R for v in vals]))


def _ints(rows):
    return c.limbs_to_ints(c.fr_from_mont(rows))


def _residues(seed, n):
    """n Montgomery residues below 2^252 from full 64-bit limbs, built without Python ints"""
    raw = np.random.default_rng(seed).integers(0, 1 << 64, (n, 4), dtype=np.uint64)
    raw[:, 3] &= (1 << 60) - 1
    return raw


def _powers_mont(x, count):
    """x^i, i < count, Montgomery rows: one block of x^i by big-int pow, then each block as the first times x^(jB)"""
    b = min(count, 1 << 13)
    base = _mont([pow(x, i, R) for i in range(b)])
    nb = -(-count // b)
    out = np.empty((nb * b, 4), dtype=np.uint64)
    step, cur = pow(x, b, R), 1
    for j in range(nb):
        out[j * b:(j + 1) * b] = c.fr_mul(base, np.broadcast_to(_mont([cur]), base.shape))
        cur = cur * step % R
    return out[:count]


def _scaled(rows, k):
    return c.fr_mul(rows, np.broadcast_to(_mont([k]), rows.shape))


def _same_rows(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got != want).reshape(len(got), -1).any(axis=1))
        pytest.fail(f"{what}: {bad.size} rows differ, the first at {bad[:8].tolist()}")


def _chain_matrices(n_vars, with_c=False):
    """synth.chain_circuit(n_vars).matrices(with_c), built with numpy (every coefficient is 1 or -1)"""
    m = n_vars - 2
    rows = np.arange(m, dtype=np.int64)
    one, neg = _mont([1]), _mont([R - 1])

    def csr(cols, v):
        return csr_from_coo(rows, cols.astype(np.uint32), np.repeat(v, m, axis=0), m)
    cm = ConstraintMatrices(2, n_vars - 2, m, m, m, 0, csr(rows + 2, neg), csr(rows + 2, one))
    if with_c:
        cm.c = csr(np.where(rows + 3 < n_vars, rows + 3, 1), neg)
        cm.c_num_non_zero = m
    return cm


def _h_circom_rows(n, tau, delta_inv, rows):
    """synth.h_query_scalars(n, tau, delta_inv)[k] for the given k only (its closed form, row by row)"""
    w = synth.root_of_unity(2 * n)
    t_top = pow(tau, 2 * n - 1, R)
    cst = delta_inv * pow(2 * n, -1, R) % R
    out = []
    for k in rows:
        wj = pow(w, 2 * int(k) + 1, R)
        out.append(cst * (t_top * wj - 1) % R * pow((tau * pow(wj, -1, R) - 1) % R, -1, R) % R)
    return out


def _rows_to_check(count, slice_, seed):
    """rows within 2 of every multiple of slice_, the first and last row, and 1024 random rows"""
    rows = {0, count - 1} | {b + d for b in range(slice_, count, slice_) for d in range(-2, 3)}
    rows |= set(np.random.default_rng(seed).integers(0, count, 1024).tolist())
    return np.array(sorted(r for r in rows if 0 <= r < count), dtype=np.int64)


def _same_key(a, b):
    for name in KEY_FIELDS:
        _same_rows(np.ascontiguousarray(getattr(a, name)), np.ascontiguousarray(getattr(b, name)), name)


def _with(pk, **fields):
    arrs = {k: getattr(pk, k) for k in KEY_FIELDS}
    arrs.update(fields)
    return ProvingKey(pk.n_vars, pk.n_public, pk.domain_size, *(arrs[k] for k in KEY_FIELDS))


# -------------------------------------------------------------------------------------------------------------------- CPU
def test_schedule_shapes():
    """the pass shapes the docstring names, from the rule restated in _schedule"""
    assert _schedule(22) == (10, [(10, 6), (16, 6)])
    assert _schedule(23) == (10, [(10, 6), (16, 7)])
    assert _schedule(24) == (10, [(10, 7), (17, 7)])
    assert _schedule(25) == (10, [(10, 5), (15, 5), (20, 5)])
    assert _schedule(26) == (10, [(10, 5), (15, 5), (20, 6)])
    assert _schedule(27) == (10, [(10, 5), (15, 6), (21, 6)])
    assert _schedule(23, maxk=5) == (10, [(10, 4), (14, 4), (18, 5)])


@pytest.mark.parametrize('log_n', [4, 11])
def test_closed_forms_match_cref(log_n):
    """the closed forms the GPU tests expect, against oracle/cref.c in full: omega is oriented as there"""
    n = 1 << log_n
    w = synth.root_of_unity(n)
    ninv = pow(n, -1, R)
    j = 3 * n // 8 + 5
    x = np.zeros((n, 4), dtype=np.uint64)
    x[0] = _mont([1])[0]
    assert _ints(c.ntt(x)) == [1] * n
    x[0] = 0
    x[j] = _mont([1])[0]
    assert _ints(c.ntt(x)) == [pow(w, j * k, R) for k in range(n)]
    assert _ints(c.ntt(x, inverse=True)) == [pow(w, -j * k, R) * ninv % R for k in range(n)]
    g = 0x1234567890abcdef
    assert _ints(_powers_mont(g, n)) == [pow(g, i, R) for i in range(n)]
    assert _ints(c.ntt(_powers_mont(g, n))) == [(pow(g, n, R) - 1) * pow(g * pow(w, k, R) - 1, -1, R) % R for k in range(n)]


def test_helpers_restate_synth():
    for n_vars in (5, 64, 1000):
        want = synth.chain_circuit(n_vars).matrices(with_c=True)
        got = _chain_matrices(n_vars, with_c=True)
        for name in ('num_instance_variables', 'num_witness_variables', 'num_constraints', 'a_num_non_zero',
                     'b_num_non_zero', 'c_num_non_zero'):
            assert getattr(got, name) == getattr(want, name), name
        for x in ('a', 'b', 'c'):
            for u, v in zip(getattr(got, x), getattr(want, x)):
                assert np.array_equal(u, v), x
    tau, dinv = 0xabcdef12345, 0x777
    assert _h_circom_rows(64, tau, dinv, range(64)) == synth.h_query_scalars(64, tau, dinv)
    assert _powers_mont(5, (1 << 13) + 3).shape == ((1 << 13) + 3, 4)
    assert _ints(_powers_mont(5, (1 << 14) + 3)[-2:]) == [pow(5, (1 << 14) + 1, R), pow(5, (1 << 14) + 2, R)]


# ------------------------------------------------------------------------------------------------------ A. NTT, 2^23-2^27
@pytest.mark.gpu
@pytest.mark.parametrize('log_n', [23, 24, 25, 26, 27])
def test_ntt_against_cref(ctx, log_n):
    a = _residues(log_n, 1 << log_n)
    for inverse in (False, True):
        got = ctx.ntt(a, inverse=inverse)
        want = c.ntt(a, inverse=inverse)
        _same_rows(got, want, f"2^{log_n} {'inverse' if inverse else 'forward'}")
        del got, want


@pytest.mark.gpu
@pytest.mark.parametrize('log_n', [23, 27])
def test_ntt_closed_forms(ctx, log_n):
    """delta at 0 -> all ones (in full); delta at j -> omega^(jk), and its inverse omega^(-jk) / n; x^i ->
    (x^n - 1) / (x omega^k - 1); at every boundary index of the schedule and 4096 random ones"""
    n = 1 << log_n
    w = synth.root_of_unity(n)
    ks = _checked_indices(log_n, log_n)
    one = _mont([1])[0]
    x = np.zeros((n, 4), dtype=np.uint64)
    x[0] = one
    got = ctx.ntt(x)
    if not (got == one).all():
        pytest.fail(f"delta at 0: rows {np.flatnonzero((got != one).any(axis=1))[:8].tolist()} are not one")
    del got
    j = 3 * n // 8 + 5
    x[0] = 0
    x[j] = one
    got = _ints(ctx.ntt(x)[ks])
    assert got == [pow(w, j * int(k), R) for k in ks], "delta at j, forward"
    ninv = pow(n, -1, R)
    got = _ints(ctx.ntt(x, inverse=True)[ks])
    assert got == [pow(w, -j * int(k), R) * ninv % R for k in ks], "delta at j, inverse"
    del x
    g = 0x5eed0000000000000000000000000000000000000000000000000000000001
    xs = _powers_mont(g, n)
    got = _ints(ctx.ntt(xs)[ks])
    del xs
    top = pow(g, n, R) - 1
    assert got == [top * pow(g * pow(w, int(k), R) - 1, -1, R) % R for k in ks], "geometric"


@pytest.mark.gpu
def test_witness_map_2p23_vs_cref(ctx):
    """both reductions at 2^23 rows (their transforms run the 2^23 schedule), on a random full assignment"""
    n_vars = 1 << 23
    cm = _chain_matrices(n_vars, with_c=True)
    w = _residues(0x23, n_vars)
    m = cm.num_constraints
    h = CircomReduction.witness_map_from_matrices(cm, 2, m, w, ctx)
    _same_rows(h, c.witness_map(m, 2, n_vars, cm.a, cm.b, w), "CircomReduction")
    del h
    h = LibsnarkReduction.witness_map_from_matrices(cm, 2, m, w, ctx)
    _same_rows(h, c.witness_map_libsnark(m, 2, cm.a, cm.b, cm.c, w), "LibsnarkReduction")
    release(cm)


@pytest.mark.gpu
@pytest.mark.parametrize('env', [dict(B2G_NTT_RADIX2='1'), dict(B2G_NTT_MAXK='5')],
                         ids=lambda e: ','.join('%s=%s' % (k[8:], v) for k, v in e.items()))
def test_ntt_2p23_pass_schedules(ctx, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    a = _residues(0x123, 1 << 23)
    for inverse in (False, True):
        _same_rows(ctx.ntt(a, inverse=inverse), c.ntt(a, inverse=inverse), f"{env} {'inverse' if inverse else 'forward'}")


# ----------------------------------------------------------------------------------------------- ceremony of power 23
class _Ceremony:
    """a ceremony of size 2^power for seeded (tau, alpha, beta) on the standard generators, by fixed-base products; the
    powers of tau are built in Montgomery rows, never as a list of Python ints"""

    def __init__(self, ctx, power, seed):
        rng = random.Random(seed)
        self.tau, self.alpha, self.beta = (rng.randrange(2, R) for _ in range(3))
        self.power = self.ceremony_power = power
        n = 1 << power
        t = _powers_mont(self.tau, 2 * n - 1)
        self.tau_g1 = ctx.fixed_base_g1(c.fr_from_mont(t))
        self.tau_g2 = ctx.fixed_base_g2(c.fr_from_mont(t[:n]))
        self.alpha_tau_g1 = ctx.fixed_base_g1(c.fr_from_mont(_scaled(t[:n], self.alpha)))
        self.beta_tau_g1 = ctx.fixed_base_g1(c.fr_from_mont(_scaled(t[:n], self.beta)))
        self.beta_g2 = ctx.fixed_base_g2(c.ints_to_limbs([self.beta]))

    def prefix(self, power):
        return Powers(power, power, *(getattr(self, k) for k in ARRAYS)).prefix(power)


@pytest.fixture(scope='module')
def cer23(ctx):
    return _Ceremony(ctx, 23, 0x2323)


# ------------------------------------------------------------------------------------------ B. setup across the slices
@pytest.mark.gpu
def test_setup_across_setup_slice(ctx):
    """2^20 + 37 variables (domain 2^21): every key array crosses SETUP_SLICE, H twice; both reductions, in full, against
    synth.setup_scalars through the fixed-base products"""
    n_vars = SETUP_SLICE + 37
    circ = synth.chain_circuit(n_vars)
    cm = _chain_matrices(n_vars, with_c=True)
    rng = random.Random(0x5E7)
    tau, alpha, beta, gamma, delta = (rng.randrange(1, R) for _ in range(5))
    td = synth.setup_scalars(circ, trapdoor=(tau, alpha, beta, gamma, delta))
    n = circ.domain_size
    assert n == 2 * SETUP_SLICE
    g1 = ctx.fixed_base_g1(synth._ints_to_limbs([alpha, beta, delta] + td.ic_t + td.a_t + td.b_t + td.l_t))
    g2 = ctx.fixed_base_g2(synth._ints_to_limbs([beta, gamma, delta] + td.b_t))
    ni = circ.num_inputs
    o = 3 + ni
    want = dict(alpha_g1=g1[0:1], beta_g1=g1[1:2], delta_g1=g1[2:3], beta_g2=g2[0:1], gamma_g2=g2[1:2], delta_g2=g2[2:3],
                gamma_abc_g1=g1[3:o], a_query=g1[o:o + n_vars], b_g1_query=g1[o + n_vars:o + 2 * n_vars],
                l_query=g1[o + 2 * n_vars:], b_g2_query=g2[3:])
    dinv = pow(delta, -1, R)
    hs = {CircomReduction: td.h_t, LibsnarkReduction: synth.h_query_scalars_libsnark(n, tau, dinv)}
    for red, h_t in hs.items():
        pk = Groth16.generate_parameters_with_qap(cm, alpha, beta, gamma, delta, tau=tau, ctx=ctx, reduction=red)
        for name, arr in want.items():
            _same_rows(getattr(pk, name), arr, f"{red.__name__} {name}")
        _same_rows(pk.h_query, ctx.fixed_base_g1(synth._ints_to_limbs(h_t)), f"{red.__name__} h_query")


@pytest.mark.gpu
def test_circom_setup_at_2p22(ctx, cer23):
    """n = 2^22: the H query comes from a 2^23 transform; its rows around every SETUP_SLICE multiple, the last and 1024
    random rows against the closed form; the key from the power-22 ceremony is byte-identical"""
    n_vars = 1 << 22
    cm = _chain_matrices(n_vars, with_c=True)
    pk = Groth16.generate_parameters_with_qap(cm, cer23.alpha, cer23.beta, 1, 1, tau=cer23.tau, ctx=ctx)
    rows = _rows_to_check(n_vars, SETUP_SLICE, 22)
    want = ctx.fixed_base_g1(synth._ints_to_limbs(_h_circom_rows(n_vars, cer23.tau, 1, rows)))
    _same_rows(np.asarray(pk.h_query)[rows], want, "h_query")
    _same_key(Groth16.generate_parameters_from_powers_of_tau(cm, cer23.prefix(22), ctx), pk)


@pytest.mark.gpu
def test_verify_proving_key_across_powers_slice(ctx, cer23):
    """2^22 + 37 variables, domain 2^23, power-23 ceremony: key arrays stream in two POWERS_SLICE pieces; a point off the
    curve on either side of the boundary and at the end is named by its index; a valid but wrong point is found"""
    n_vars = POWERS_SLICE + 37
    cm = _chain_matrices(n_vars, with_c=True)
    pk = Groth16.generate_parameters_with_qap(cm, cer23.alpha, cer23.beta, 1, 1, tau=cer23.tau, ctx=ctx)
    assert pk.domain_size == 1 << 23
    r = Groth16.verify_proving_key(cm, cer23, pk, ctx=ctx)
    assert r and r.reason is None, r.reason
    for i in (POWERS_SLICE - 1, POWERS_SLICE, n_vars - 1):
        a = np.array(pk.a_query, copy=True)
        assert a[i].any()
        a[i, 4] ^= 1
        r = Groth16.verify_proving_key(cm, cer23, _with(pk, a_query=a), ctx=ctx)
        assert not r and r.reason == f'a_query[{i}]: off the curve', (i, r.reason)
    a = np.array(pk.a_query, copy=True)
    a[POWERS_SLICE] = ctx.test_op(10, a[POWERS_SLICE])[0]
    r = Groth16.verify_proving_key(cm, cer23, _with(pk, a_query=a), ctx=ctx)
    assert not r and r.reason == 'a_query does not match the circuit and ceremony', r.reason


# ------------------------------------------------------------------------------------- C. preparation across PREP_PINNED
@pytest.mark.gpu
def test_prepare_across_the_pinned_buffer(ctx, cer23, tmp_path):
    """power 20: tau_g1 block 21 and tau_g2 block 20 are two pinned pieces each, tau_g1 block 20 exactly one; against the
    inverse point transform of the ceremony's points (b2g_points_intt, which does not go through to_host); then the same
    into a memory-mapped file, read back with its Lagrange sections"""
    assert (2 << 20) * 64 == 2 * PREP_PINNED and (1 << 20) * 128 == 2 * PREP_PINNED and (1 << 20) * 64 == PREP_PINNED
    got = Groth16.prepare_powers_of_tau(cer23, power=20, ctx=ctx)
    assert got.power == 20 and got.lagrange.power == 20
    for name, blocks, g2 in (('tau_g1', (19, 20, 21), False), ('tau_g2', (19, 20), True)):
        mono, lag = getattr(cer23, name), getattr(got.lagrange, name)
        for k in blocks:
            m = 1 << k
            src = mono[:m] if k <= 20 else np.concatenate([mono[:m - 1], np.zeros((1, 8), dtype=np.uint64)])
            _same_rows(lag[m - 1:2 * m - 1], ctx.points_intt(src, g2=g2), f"{name} block {k}")
    path = tmp_path / 'pot20_prepared.ptau'
    Groth16.prepare_powers_of_tau(cer23, dst=str(path), power=20, ctx=ctx)
    back = read_ptau(str(path))
    assert back.power == 20 and back.lagrange is not None and back.lagrange.power == 20
    for name in LAGRANGE:
        _same_rows(getattr(back.lagrange, name), getattr(got.lagrange, name), f"file lagrange_{name}")
    for name in ARRAYS:
        _same_rows(getattr(back, name), getattr(got, name), f"file {name}")


# ---------------------------------------------------------------------------------- D. key serialization across KEY_SLICE
def _ser(ctx, pts, g2, compress):
    pts = np.ascontiguousarray(pts, dtype='<u8')
    n = len(pts)
    out = np.zeros(n * M.point_size(g2, compress), dtype=np.uint8)
    N.check(N.lib().b2g_points_serialize(ctx._h, int(g2), int(compress), n, pts.ctypes.data, out.ctypes.data))
    return out


def _de(ctx, raw, g2, compress):
    """(points, the first refused index or the count)"""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n = raw.size // M.point_size(g2, compress)
    pts = np.zeros((n, 16 if g2 else 8), dtype='<u8')
    first = C.c_uint64()
    N.check(N.lib().b2g_points_deserialize(ctx._h, int(g2), int(compress), n, raw.ctypes.data, pts.ctypes.data, C.byref(first)))
    return pts, first.value


@pytest.fixture(scope='module')
def key_points(ctx):
    """2^20 + 5 G1 and G2 points of random scalars, with infinity on both sides of the slice"""
    n = KEY_SLICE + 5
    sc = _residues(0x5E, n)
    sc[[3, KEY_SLICE - 3, KEY_SLICE + 1]] = 0
    return {False: ctx.fixed_base_g1(sc), True: ctx.fixed_base_g2(sc)}


@pytest.mark.gpu
@pytest.mark.parametrize('compress', [True, False])
@pytest.mark.parametrize('g2', [False, True], ids=['g1', 'g2'])
def test_points_serialization_across_key_slice(ctx, key_points, g2, compress):
    """one call on 2^20 + 5 points equals the two single-slice calls on [0, 2^20) and [2^20, end), both directions; the
    rows at the boundary and the last are the big-int model's bytes"""
    pts, s = key_points[g2], KEY_SLICE
    size = M.point_size(g2, compress)
    whole = _ser(ctx, pts, g2, compress)
    _same_rows(whole.reshape(-1, size), np.concatenate([_ser(ctx, pts[:s], g2, compress),
                                                         _ser(ctx, pts[s:], g2, compress)]).reshape(-1, size), "serialized")
    for i in (s - 3, s - 2, s - 1, s, s + 1, s + 4):
        pt = V._g2_from_words(pts[i]) if g2 else V._g1_from_words(pts[i])
        assert whole[i * size:(i + 1) * size].tobytes() == M.point_bytes(pt, g2, compress), i
    got, first = _de(ctx, whole, g2, compress)
    assert first == len(pts)
    _same_rows(got, pts, "deserialized")
    lo, f0 = _de(ctx, whole[:s * size], g2, compress)
    hi, f1 = _de(ctx, whole[s * size:], g2, compress)
    assert (f0, f1) == (s, len(pts) - s)
    _same_rows(got, np.concatenate([lo, hi]), "deserialized in two calls")


def _bad_points(pts, i, g2, compress):
    """{kind: bytes of one bad point} from the valid point i"""
    x, y = V._g2_from_words(pts[i]) if g2 else V._g1_from_words(pts[i])
    out = {}
    above = bytearray(M.point_bytes((x, y), g2, compress))
    above[:32] = P.to_bytes(32, 'little')                # x (x.c0 in G2) = p
    out['coordinate >= p'] = bytes(above)
    if compress:
        out['off the curve'] = g2_bytes(g2_no_root_x()) if g2 else g1_no_root_x().to_bytes(32, 'little')
    else:
        out['off the curve'] = bytes(M._le([x[0], x[1], (y[0] + 1) % P, y[1]] if g2 else [x, (y + 1) % P]))
    if g2:
        out['outside G2'] = M.point_bytes(twist_point_outside_g2(random.Random(5)), True, compress)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('compress', [True, False])
@pytest.mark.parametrize('g2', [False, True], ids=['g1', 'g2'])
def test_refusals_across_key_slice(ctx, key_points, g2, compress):
    """a bad point at 2^20 - 1, 2^20 or 2^20 + 4 is refused with its absolute index; of two, the lower one is reported"""
    pts, s = key_points[g2], KEY_SLICE
    size = M.point_size(g2, compress)
    whole = _ser(ctx, pts, g2, compress)
    at = (s - 1, s, s + 4)
    for i in at:
        for kind, raw in _bad_points(pts, i, g2, compress).items():
            data = whole.copy()
            data[i * size:(i + 1) * size] = np.frombuffer(raw, dtype=np.uint8)
            assert _de(ctx, data, g2, compress)[1] == i, (i, kind)
    for pair in ((s - 1, s + 4), (s, s + 4)):
        data = whole.copy()
        for i in pair:
            data[i * size:(i + 1) * size] = np.frombuffer(_bad_points(pts, i, g2, compress)['off the curve'], dtype=np.uint8)
        assert _de(ctx, data, g2, compress)[1] == pair[0], pair
    for i in at:                                          # the writer's refusal of a Montgomery coordinate >= p
        bad = np.array(pts, copy=True)
        bad[i, :4] = np.frombuffer(P.to_bytes(32, 'little'), dtype='<u8')
        with pytest.raises(N.B2gError, match=f'point {i} has a coordinate >= p'):
            _ser(ctx, bad, g2, compress)
