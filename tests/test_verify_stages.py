"""Each device verifier stage against the big-int pairing model (oracle/pairing_model.py) and the host verifier
(circom_compat_b200/verifier.py), at the values where a tower, loop or table kernel goes wrong: zero, one, -1, sparse and
subfield elements, coordinates p - 1 and p - 2, the degenerate line steps, every Miller-loop instantiation, the prepared
lines, the public-input window tables and keys whose IC points coincide, cancel or are infinity, and proof points B of small
order outside G2.  Tower and loop results are compared as raw Montgomery words, so a result that is right modulo p but not
reduced below p fails too."""
import random

import numpy as np
import pytest

from batch_model import g2_in_subgroup, twist_point_outside_g2
from circom_compat_b200 import verifier as V
from oracle import pairing_model as M
from oracle import pyref as o

pytestmark = pytest.mark.gpu

P, R = V.P, o.R_MOD
_RM = 1 << 256
_RM_INV = pow(_RM, -1, P)
F2_ZERO, F2_ONE = V.F2_ZERO, V.F2_ONE
F12_ZERO = ((F2_ZERO,) * 3,) * 2
F12_MINUS_ONE = (((P - 1, 0), F2_ZERO, F2_ZERO), (F2_ZERO,) * 3)
# the twist's order r (2p - r) and the small primes of its cofactor 2p - r (the fourth one has 177 bits)
TWIST_ORDER = R * (2 * P - R)
SMALL_ORDERS = (10069, 5864401, 1875725156269)


# ---------------------------------------------------------------------------------------------- encodings
def _words(vals):
    """canonical integers -> Montgomery 64-bit words, 4 per value"""
    return np.frombuffer(b''.join((v * _RM % P).to_bytes(32, 'little') for v in vals), dtype='<u8').copy()


def _rows(rows_of_vals):
    return np.stack([_words(vals) for vals in rows_of_vals])


def _f12_vals(f):
    return [c for f6 in f for f2 in f6 for c in f2]


def _f12_rows(fs):
    return _rows([_f12_vals(f) for f in fs])


def _f2_vals(xs):
    return [c for x in xs for c in x]


def _g1_vals(p):
    return [0, 0] if p is None else list(p)


def _g2_vals(q):
    return [0] * 4 if q is None else [q[0][0], q[0][1], q[1][0], q[1][1]]


def _ints(row):
    raw = np.ascontiguousarray(row, dtype='<u8').tobytes()
    return [int.from_bytes(raw[i:i + 32], 'little') * _RM_INV % P for i in range(0, len(raw), 32)]


def _xyzz_affine(row):
    x, y, zz, zzz = _ints(row)
    if zz == 0:
        return None
    return (x * pow(zz, -1, P) % P, y * pow(zzz, -1, P) % P)


def _g1(k):
    return o.G1.mul(o.G1_GEN, k)


def _g2(k):
    return o.G2.mul(o.G2_GEN, k)


def _proof(a, b, c):
    from circom_compat_b200 import Proof
    return Proof(b''.join(int(v).to_bytes(32, 'little') for v in _g1_vals(a) + _g2_vals(b) + _g1_vals(c)))


def _assert_rows(got, want, what):
    """raw word equality, naming the first row that differs"""
    assert got.shape == want.shape, what
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{what}: {bad.size} of {len(want)} rows differ, first at row {bad[0]}"


# ---------------------------------------------------------------------------------------------- structured Fq12 values
def _residue_pool(rng):
    """Fq values with extreme limb patterns (as in test_gpu_parity's raw residues), reduced below p"""
    pat = [0, 1, 0xffffffff, 0xfffffffe, 0x80000000, 0x7fffffff]
    out = [0, 1, 2, P - 1, P - 2, P - 3, P >> 1, (P + 1) >> 1, (1 << 253) - 1, 1 << 253, (1 << 254) % P, _RM % P, (-_RM) % P]
    for _ in range(40):
        out.append(sum(rng.choice(pat + [rng.getrandbits(32)]) << (32 * i) for i in range(8)) % P)
    return out


def _structured_f12(rng, n):
    """n Fq12 values: the fixed edge values, then elements whose coordinates come from the residue pool or are random,
    with a random sparsity: only c0, only c1, a single Fq2 slot, Fq or Fq2 embedded, every coordinate p - 1, or p - 1 and
    p - 2 alternating (so the Karatsuba operand sums reach 2p - 3)"""
    pool = _residue_pool(rng)
    fixed = [F12_ZERO, V.F12_ONE, F12_MINUS_ONE,
             ((( P - 1, P - 1),) * 3,) * 2,
             (((P - 1, P - 2),) * 3,) * 2,
             (((P - 2, P - 1),) * 3,) * 2,
             (((P - 2, P - 2),) * 3,) * 2,
             ((F2_ZERO,) * 3, (F2_ONE, F2_ZERO, F2_ZERO)),                    # w
             ((F2_ZERO, F2_ONE, F2_ZERO), (F2_ZERO,) * 3),                    # v
             (((0, 1), F2_ZERO, F2_ZERO), (F2_ZERO,) * 3)]                    # u
    for slot in range(6):                                                    # one slot at p - 1 (both) and 1
        for v in ((P - 1, P - 1), (1, 0), (0, 1)):
            c = [F2_ZERO] * 6
            c[slot] = v
            fixed.append((tuple(c[:3]), tuple(c[3:])))
    out = list(fixed)
    while len(out) < n:
        kind = rng.randrange(8)
        coord = (lambda: rng.choice(pool)) if rng.random() < 0.6 else (lambda: rng.randrange(P))
        c = [(coord(), coord()) for _ in range(6)]
        if kind == 0:
            c[3:] = [F2_ZERO] * 3                                            # only c0
        elif kind == 1:
            c[:3] = [F2_ZERO] * 3                                            # only c1
        elif kind == 2:
            keep = rng.randrange(6)
            c = [x if k == keep else F2_ZERO for k, x in enumerate(c)]       # one Fq2 slot
        elif kind == 3:
            c = [(c[0][0], 0)] + [F2_ZERO] * 5                               # Fq
        elif kind == 4:
            c = [c[0]] + [F2_ZERO] * 5                                       # Fq2
        elif kind == 5:
            c = [(P - 1, P - 2) if rng.random() < 0.5 else (P - 2, P - 1) for _ in range(6)]
        elif kind == 6:
            c = [x if rng.random() < 0.5 else F2_ZERO for x in c]            # random zero slots
        out.append((tuple(c[:3]), tuple(c[3:])))
    return out[:n]


def _easy_part(x):
    g = V.f12_mul(V.f12_conj(x), V.f12_inv(x))
    return V.f12_mul(M.frobenius(g, 2), g)


@pytest.fixture(scope='module')
def miller_values():
    rng = random.Random(401)
    return [M.miller_loop([(_g1(rng.randrange(1, R)), _g2(rng.randrange(1, R)))]) for _ in range(4)]


@pytest.fixture(scope='module')
def cyclotomic(miller_values):
    """1, e(alpha, beta) of a key, its Frobenius images and conjugate, then the easy part of structured elements"""
    rng = random.Random(402)
    e = M.final_exponentiation(M.miller_loop([(_g1(rng.randrange(1, R)), _g2(rng.randrange(1, R)))]))
    out = [V.F12_ONE, e, V.f12_conj(e)] + [M.frobenius(e, k) for k in (1, 2, 3)] + [_easy_part(m) for m in miller_values]
    out += [_easy_part(x) for x in _structured_f12(rng, 1200) if x != F12_ZERO]    # zero has no easy part
    return out


# ---------------------------------------------------------------------------------------------- 1. tower ops
def test_fq12_products_at_structured_values(ctx, miller_values):
    rng = random.Random(300)
    xs = _structured_f12(rng, 70) + miller_values
    pairs = [(x, y) for x in xs for y in xs]
    rng.shuffle(pairs)
    pairs = pairs[:3000]
    a, b = _f12_rows([x for x, _ in pairs]), _f12_rows([y for _, y in pairs])
    _assert_rows(ctx.test_op(30, a, b), _f12_rows([V.f12_mul(x, y) for x, y in pairs]), 'op 30')
    ys = _structured_f12(random.Random(301), 3000) + miller_values
    _assert_rows(ctx.test_op(31, _f12_rows(ys)), _f12_rows([V.f12_mul(y, y) for y in ys]), 'op 31')
    for k, op in ((1, 33), (2, 34), (3, 35)):
        _assert_rows(ctx.test_op(op, _f12_rows(ys)), _f12_rows([M.frobenius(y, k) for y in ys]), f'op {op}')


def test_fq12_inverse_at_structured_values(ctx, miller_values):
    """every nonzero element against the big-int inverse; the inverse of zero is pinned as zero"""
    xs = _structured_f12(random.Random(380), 3000) + miller_values
    assert xs[0] == F12_ZERO
    want = [F12_ZERO if x == F12_ZERO else V.f12_inv(x) for x in xs]
    _assert_rows(ctx.test_op(38, _f12_rows(xs)), _f12_rows(want), 'op 38')


def test_sparse_line_product_with_zero_slots(ctx, miller_values):
    rng = random.Random(390)
    pool = _residue_pool(rng)
    xs = _structured_f12(rng, 3000) + miller_values
    choices = [F2_ZERO, F2_ONE, (P - 1, P - 1), (P - 1, P - 2), None, None]
    lines = []
    for _ in xs:
        lines.append(tuple(c if c is not None else ((rng.choice(pool), rng.randrange(P)) if rng.random() < 0.5 else
                                                    (rng.randrange(P), rng.randrange(P)))
                           for c in (rng.choice(choices) for _ in range(3))))
    want = [V.f12_mul(x, ((l[0], F2_ZERO, F2_ZERO), (l[1], l[2], F2_ZERO))) for x, l in zip(xs, lines)]
    _assert_rows(ctx.test_op(39, _f12_rows(xs), _rows([_f2_vals(l) for l in lines])), _f12_rows(want), 'op 39')


def test_cyclotomic_square_and_exponent(ctx, cyclotomic):
    want = [M.cyclotomic_sqr(g) for g in cyclotomic]
    assert want[:40] == [V.f12_mul(g, g) for g in cyclotomic[:40]]                  # the model squares cyclotomic values
    _assert_rows(ctx.test_op(32, _f12_rows(cyclotomic)), _f12_rows(want), 'op 32')
    rng = random.Random(450)
    big = [0, 1, R - 1, R, (1 << 256) - 1, 1 << 255, rng.getrandbits(256)]
    ks = [big[i] if i < len(big) else (rng.getrandbits(256) if i % 25 == 0 else rng.getrandbits(rng.choice((1, 2, 5, 12))))
          for i in range(len(cyclotomic))]
    ew = np.frombuffer(b''.join(k.to_bytes(32, 'little') for k in ks), dtype='<u8').reshape(len(ks), 4).copy()
    want = [V.f12_pow(g, k) for g, k in zip(cyclotomic, ks)]
    _assert_rows(ctx.test_op(45, _f12_rows(cyclotomic), ew), _f12_rows(want), 'op 45')


def test_final_exponentiation_at_structured_values(ctx, miller_values):
    """about fifty values; zero is pinned as zero, so a zero Miller value can never equal e(alpha, beta)"""
    xs = _structured_f12(random.Random(360), 44) + miller_values
    assert xs[0] == F12_ZERO
    want = [F12_ZERO if x == F12_ZERO else M.final_exponentiation(x) for x in xs]
    assert want[1] == want[2] == V.F12_ONE                                           # 1 and -1
    _assert_rows(ctx.test_op(36, _f12_rows(xs)), _f12_rows(want), 'op 36')


# ---------------------------------------------------------------------------------------------- 2. Miller loop shapes
def _key_points(test_zkey_bytes):
    from circom_compat_b200 import read_zkey, release
    pk, _ = read_zkey(test_zkey_bytes)
    vk = V.VerifyingKey.from_proving_key(pk)
    release(pk)
    return vk


def test_prepared_lines_match_prepare_g2(ctx, test_zkey_bytes):
    """op 50 runs vk_lines_kernel, which prepares the lines of -gamma and -delta; an odd count leaves one launch half used"""
    rng = random.Random(500)
    vk = _key_points(test_zkey_bytes)
    qs = [vk.gamma_g2, vk.delta_g2, o.G2_GEN, vk.beta_g2, _g2(rng.randrange(1, R)), twist_point_outside_g2(rng),
          _g2(rng.randrange(1, R))]
    got = ctx.test_op(50, _rows([_g2_vals(q) for q in qs]))
    want = _rows([[v for line in M.prepare_g2(V.g2_neg(q)) for v in _f2_vals(line)] for q in qs])
    _assert_rows(got, want, 'op 50')


def _xyzz_vals(p, z):
    """an affine G1 point (None = infinity) as XYZZ with ZZ = z^2, ZZZ = z^3"""
    if p is None:
        return [0] * 4
    zz, zzz = z * z % P, z * z * z % P
    return [p[0] * zz % P, p[1] * zzz % P, zz, zzz]


def test_verify_miller_kernel_every_shape(ctx, test_zkey_bytes, golden):
    """op 49 launches verify_miller_kernel on one record with lines from vk_lines_kernel: every (V_ON, NFIX) shape, reached
    as verify_many reaches it (A, B, the prepared inputs, C, gamma or delta at infinity), on random points and on a golden
    proof against its key"""
    from circom_compat_b200 import Groth16, Proof
    rng = random.Random(490)
    vk = _key_points(test_zkey_bytes)
    pvk = Groth16.process_vk(vk)
    g = golden['test_zkey']
    proof = Proof(bytes.fromhex(g['proofs'][0]['proof_hex']))
    a, b, c = V._proof_points(proof)
    prep = V.prepare_inputs(pvk, [int(x) for x in g['witness'][1:len(vk.gamma_abc_g1)]])
    rp = lambda: _g1(rng.randrange(1, R))
    rq = lambda: _g2(rng.randrange(1, R))
    cases = []                                                   # (A, B, prepared inputs, C, gamma, delta)
    for stepped in ('on', 'A = O', 'B = O'):
        for fixed in ('both', 'prep = O', 'C = O', 'gamma = O', 'delta = O', 'prep = delta = O', 'C = gamma = O', 'none'):
            pa, pb = (None if stepped == 'A = O' else rp()), (None if stepped == 'B = O' else rq())
            pr, pc, ga, de = rp(), rp(), rq(), rq()
            if 'prep' in fixed or fixed == 'none': pr = None
            if fixed.startswith('C') or fixed == 'none': pc = None
            if 'gamma' in fixed: ga = None
            if 'delta' in fixed: de = None
            cases.append((pa, pb, pr, pc, ga, de))
    cases.append((a, b, prep, c, vk.gamma_g2, vk.delta_g2))
    cases.append((None, None, prep, c, vk.gamma_g2, vk.delta_g2))
    cases.append((a, b, None, c, vk.gamma_g2, None))
    rows = _rows([_g1_vals(pa) + _g2_vals(pb) + _g1_vals(pr) + _g1_vals(pc) + _g2_vals(ga) + _g2_vals(de)
                  for pa, pb, pr, pc, ga, de in cases])
    got = ctx.test_op(49, rows)
    want = [M.miller_loop([(pa, pb), (pr, V.g2_neg(ga)), (pc, V.g2_neg(de))]) for pa, pb, pr, pc, ga, de in cases]
    _assert_rows(got, _f12_rows(want), 'op 49')
    # the golden proof's whole Miller value: its final exponentiation is e(alpha, beta)
    assert M.final_exponentiation(want[-3]) == pvk.alpha_g1_beta_g2


def test_batch_pairs_kernel_every_shape(ctx, test_zkey_bytes):
    """op 53 launches batch_pairs_kernel on a tail holding the prepared inputs and sum r C as XYZZ points with Z != 1:
    two, one or no prepared pairs, dropped by a point or by gamma or delta at infinity"""
    rng = random.Random(530)
    vk = _key_points(test_zkey_bytes)
    rp = lambda: _g1(rng.randrange(1, R))
    rq = lambda: _g2(rng.randrange(1, R))
    cases = [(rp(), rp(), rq(), rq()), (rp(), rp(), vk.gamma_g2, vk.delta_g2), (None, rp(), rq(), rq()),
             (rp(), None, rq(), rq()), (rp(), rp(), None, rq()), (rp(), rp(), rq(), None), (None, None, rq(), rq()),
             (rp(), rp(), None, None), (rp(), None, rq(), None), (o.G1_GEN, o.G1_GEN, o.G2_GEN, o.G2_GEN)]
    rows = _rows([_xyzz_vals(pr, rng.randrange(2, P)) + _xyzz_vals(pc, rng.randrange(2, P)) + _g2_vals(ga) + _g2_vals(de)
                  for pr, pc, ga, de in cases])
    got = ctx.test_op(53, rows)
    want = [M.miller_loop([(pr, V.g2_neg(ga)), (pc, V.g2_neg(de))]) for pr, pc, ga, de in cases]
    _assert_rows(got, _f12_rows(want), 'op 53')


# ---------------------------------------------------------------------------------------------- 3. degenerate line steps
def _proj(q, z):
    return (V.f2_mul(q[0], z), V.f2_mul(q[1], z), z)


def test_degenerate_line_steps_match_the_model(ctx):
    rng = random.Random(410)
    rz = lambda: (rng.randrange(1, P), rng.randrange(P))
    q = _g2(rng.randrange(1, R))
    # the twist has no point with y = 0 (its order is odd) and none with x = 0 (b' is not a square in Fq2)
    assert TWIST_ORDER % 2 == 1
    y0 = o._fq2_sqrt(V.TWIST_B)
    assert y0 is None or V.f2_sqr(y0) != V.TWIST_B
    assert pow(V.TWIST_B[0] ** 2 + V.TWIST_B[1] ** 2, (P - 1) // 2, P) == P - 1           # its norm is not a square in Fq
    far = twist_point_outside_g2(rng)
    ts = [(F2_ZERO, F2_ONE, F2_ZERO), (rz(), rz(), F2_ZERO), (F2_ZERO, F2_ZERO, F2_ZERO), (F2_ONE, F2_ZERO, F2_ONE),
          _proj(q, rz()), _proj(V.g2_neg(q), rz()), _proj(far, rz())]
    dbl = ctx.test_op(41, _rows([_f2_vals(t) for t in ts]))
    _assert_rows(dbl, _rows([_f2_vals(t2 + l) for t2, l in (M.dbl_step(t) for t in ts)]), 'op 41')
    cases = [((F2_ZERO, F2_ONE, F2_ZERO), q), ((rz(), rz(), F2_ZERO), q),                       # T with Z = 0
             (_proj(q, rz()), q), (_proj(q, F2_ONE), q),                                        # T = Q
             (_proj(V.g2_neg(q), rz()), q), (_proj(V.g2_neg(q), F2_ONE), q),                    # T = -Q
             (_proj(far, rz()), far), (_proj(V.g2_neg(far), rz()), far),
             (_proj(q, rz()), (F2_ZERO, F2_ZERO))]                                              # Q given as zeros
    add = ctx.test_op(42, _rows([_f2_vals(t) for t, _ in cases]), _rows([_f2_vals(q_) for _, q_ in cases]))
    _assert_rows(add, _rows([_f2_vals(t2 + l) for t2, l in (M.add_step(t, q_) for t, q_ in cases)]), 'op 42')


# ---------------------------------------------------------------------------------------------- 4. window tables, prepared inputs
def test_window_table_rows(ctx):
    """all 32 x 255 rows of the table of a G1 point (and the all-zero table of infinity) against repeated addition"""
    p = _g1(random.Random(520).randrange(1, R))
    got = ctx.test_op(52, _rows([_g1_vals(p), _g1_vals(None)]))
    want = []
    base = p
    for _ in range(32):
        acc = None
        for _ in range(255):
            acc = V.g1_add(acc, base)
            want.append(acc)
        base = V.g1_add(acc, base)                                               # 256 * base
    assert got[0].tobytes() == _words([v for q in want for v in q]).tobytes()
    assert not got[1].any()


def test_window_table_product(ctx):
    """x P through the public-input kernel on a table: one digit per lane at 0x01, 0x80 and 0xff, 2^(8k), all-0xff bytes,
    r - 1, and values below 2^64 and 2^160"""
    rng = random.Random(510)
    ks = [0, 1, 2, 255, 256, R - 1, R - 2, (R - 1) // 2, (1 << 256) - 1, (1 << 64) - 1, (1 << 160) - 1]
    ks += [d << (8 * lane) for lane in range(32) for d in (0x01, 0x80, 0xff)]
    ks += [int.from_bytes(bytes(rng.choice((0, 1, 0xff)) for _ in range(32)), 'little') for _ in range(40)]
    ks += [rng.getrandbits(64) for _ in range(10)] + [rng.getrandbits(160) for _ in range(10)] + [rng.randrange(R) for _ in range(10)]
    kw = np.frombuffer(b''.join(k.to_bytes(32, 'little') for k in ks), dtype='<u8').reshape(len(ks), 4).copy()
    for p in (o.G1_GEN, _g1(rng.randrange(1, R))):
        got = [_xyzz_affine(r) for r in ctx.test_op(51, kw, _words(_g1_vals(p)))]
        want = [o.G1.mul(p, k) for k in ks]
        bad = [k for k, g, w in zip(ks, got, want) if g != w]
        assert not bad, f"{len(bad)} scalars differ, first {bad[0]:#x}"
    got = ctx.test_op(51, kw[:4], _words([0, 0]))                                # the table of infinity
    assert [_xyzz_affine(r) for r in got] == [None] * 4


def _edge_key(seed, n_public, ic_logs):
    """a key with known discrete logs; ic_logs maps an IC index to its log (0: infinity), the others are random"""
    rng = random.Random(seed)
    al, be, ga, de = (rng.randrange(1, R) for _ in range(4))
    ic = [ic_logs(j, rng) for j in range(n_public + 1)]
    vk = V.VerifyingKey(_g1(al), _g2(be), _g2(ga), _g2(de), [_g1(k) if k % R else None for k in ic])
    return vk, (al, be, ga, de), ic, rng


def _proofs_for(logs, ic, rng, inputs_list):
    """a valid proof per inputs, then each one with C + G (invalid)"""
    al, be, ga, de = logs
    valid = []
    for xs in inputs_list:
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        prep = (ic[0] + sum(x * k for x, k in zip(xs, ic[1:]))) % R
        c = (a * b - al * be - prep * ga) * pow(de, -1, R) % R
        valid.append(_proof(_g1(a), _g2(b), _g1(c)))
    bad = [_proof(V._proof_points(p)[0], V._proof_points(p)[1], o.G1.add(V._proof_points(p)[2], o.G1_GEN)) for p in valid]
    return valid, bad


def _edge_keys():
    """(name, vk, logs, ic, rng, inputs for verify_many, inputs for verify_batch)"""
    out = []
    vk, logs, ic, rng = _edge_key(600, 0, lambda j, r: 0)                                  # the only IC at infinity
    out.append(('n=0, IC[0] = O', vk, logs, ic, rng, [[], []], [[], [], []]))
    vk, logs, ic, rng = _edge_key(601, 0, lambda j, r: r.randrange(1, R))
    out.append(('n=0', vk, logs, ic, rng, [[], []], [[], [], []]))
    vk, logs, ic, rng = _edge_key(602, 1, lambda j, r: 0 if j == 1 else r.randrange(1, R))   # x O
    out.append(('n=1, IC[1] = O', vk, logs, ic, rng, [[5], [R - 1]], [[0], [1], [R - 1]]))
    vk, logs, ic, rng = _edge_key(603, 1, lambda j, r: r.randrange(1, R))
    out.append(('n=1', vk, logs, ic, rng, [[0], [R - 1]], [[1], [rng.randrange(R)], [0]]))
    q = random.Random(604).randrange(1, R)
    # IC[0] = O and IC[1] = IC[2]: equal inputs double in the sequential sum and in the tree sum
    vk, logs, ic, rng = _edge_key(605, 2, lambda j, r: 0 if j == 0 else q)
    x = rng.randrange(R)
    out.append(('IC[0] = O, IC[1] = IC[2]', vk, logs, ic, rng, [[x, x], [R - 1, R - 1]], [[x, x], [1, 1], [7, 7]]))
    # IC[0] = k IC[1], IC[1] = IC[2]: IC[0] + x1 IC[1] = x2 IC[2] when x2 = x1 + k (verify_many's running sum), and
    # s_0 IC[0] + s_2 IC[2] = s_1 IC[1] when x1 = x2 + k for every proof (verify_batch's tree: (0 + 2) + 1)
    k = random.Random(606).randrange(1, R)
    vk, logs, ic, rng = _edge_key(607, 2, lambda j, r: k * q % R if j == 0 else q)
    out.append(('IC[0] = k IC[1], IC[1] = IC[2]', vk, logs, ic, rng, [[3, (3 + k) % R], [R - 1, (k - 1) % R]],
                [[(5 + k) % R, 5], [k, 0], [(k - 1) % R, R - 1]]))
    # IC[2] = -IC[1] with equal inputs: the two terms cancel (to infinity when IC[0] = O, which drops the gamma pair)
    for name, ic0 in (('IC[0] = O, IC[2] = -IC[1]', 0), ('IC[2] = -IC[1]', 1)):
        vk, logs, ic, rng = _edge_key(608 + ic0, 2, lambda j, r: (r.randrange(1, R) if ic0 else 0) if j == 0 else (q if j == 1 else R - q))
        x = rng.randrange(R)
        out.append((name, vk, logs, ic, rng, [[x, x], [1, 1]], [[x, x], [2, 2], [R - 1, R - 1]]))
    # 130 inputs: an IC at infinity, two equal, two opposite; 0, 1 and r - 1 away from position 0
    def ic130(j, r):
        return {5: 0, 8: q, 9: q, 10: q, 11: R - q}.get(j, r.randrange(1, R))
    vk, logs, ic, rng = _edge_key(610, 130, ic130)
    xs = [[rng.choice((0, 1, R - 1, rng.randrange(R))) for _ in range(130)] for _ in range(3)]
    for v in xs:
        v[7], v[8], v[9], v[10] = v[8], v[8], v[9], v[9]                          # IC[8] = IC[9]; IC[10] = -IC[11]
    out.append(('n=130', vk, logs, ic, rng, xs[:2], xs))
    return out


def test_prepared_inputs_edge_keys(ctx):
    """verify_many against the host verifier and verify_batch on keys with 0, 1, 2 and 130 inputs whose IC points are
    infinity, equal or opposite"""
    from circom_compat_b200 import Groth16, release
    for name, vk, logs, ic, rng, many_inputs, batch_inputs in _edge_keys():
        pvk = V.prepare_verifying_key(vk)
        valid, bad = _proofs_for(logs, ic, rng, many_inputs)
        inputs, proofs = many_inputs + many_inputs, valid + bad
        want = [V.verify_with_processed_vk(pvk, xs, p) for xs, p in zip(inputs, proofs)]
        assert want == [True] * len(valid) + [False] * len(bad), name
        assert Groth16.verify_many(vk, inputs, proofs, ctx) == want, name
        bvalid, bbad = _proofs_for(logs, ic, rng, batch_inputs)
        assert Groth16.verify_batch(vk, batch_inputs, bvalid, ctx), name
        assert not Groth16.verify_batch(vk, batch_inputs, bvalid[:-1] + bbad[-1:], ctx), name
        release(vk)


# ---------------------------------------------------------------------------------------------- 5. B of small order
def _g2_mul_raw(pt, k):
    """k pt on the twist without reducing k modulo r"""
    F = o.FQ2
    acc, base = o._to_jac(F, None), o._to_jac(F, pt)
    for bit in bin(k)[2:]:
        acc = o._jac_double(F, acc)
        if bit == '1':
            acc = o._jac_add(F, acc, base)
    return o._to_affine(F, acc)


@pytest.fixture(scope='module')
def small_order_points():
    """per small prime q of the twist cofactor: a point S of order q, and G + S for a G2 point G"""
    rng = random.Random(700)
    out = []
    for q in SMALL_ORDERS:
        while True:
            s = _g2_mul_raw(twist_point_outside_g2(rng), TWIST_ORDER // q)
            if s is not None:
                break
        assert _g2_mul_raw(s, q) is None and V.g2_on_curve(s)
        out += [(q, s), (q, o.G2.add(_g2(rng.randrange(1, R)), s))]
    return out


def _affine_walk_is_regular(b) -> bool:
    """whether an affine Miller loop on b (the host verifiers' loops, Python and C++) divides by zero nowhere: no doubling of
    a point with y = 0, no addition of T and Q with x_T = x_Q (T = -Q, or T = Q, which the host lines treat as a doubling,
    but their chord branch would not), and T never infinity, through the 65 digits and both Frobenius steps"""
    t, nb = b, V.g2_neg(b)
    steps = []
    for d in M.ATE_NAF[1:]:
        steps.append(None)
        if d:
            steps.append(b if d == 1 else nb)
    steps += [M.twist_frobenius(b), M.twist_frobenius2_neg(b)]
    for q in steps:
        if q is None:
            if t[1] == F2_ZERO:
                return False
            t = o.G2.add(t, t)
        else:
            if t[0] == q[0]:
                return False
            t = o.G2.add(t, q)
        if t is None:
            return False
    return True


def test_small_order_b_values(ctx, small_order_points):
    """the Miller value and the pairing of (P, B) for B of small order, or a G2 point plus one, equal the model's"""
    rng = random.Random(701)
    qs = [b for _, b in small_order_points]
    ps = [_g1(rng.randrange(1, R)) for _ in qs]
    got = ctx.test_op(40, _rows([_g1_vals(p) for p in ps]), _rows([_g2_vals(b) for b in qs]))
    _assert_rows(got, _f12_rows([M.miller_loop([(p, b)]) for p, b in zip(ps, qs)]), 'op 40')
    got = ctx.test_op(37, _rows([_g1_vals(p) for p in ps]), _rows([_g2_vals(b) for b in qs]))
    _assert_rows(got, _f12_rows([M.pairing(p, b) for p, b in zip(ps, qs)]), 'op 37')
    assert [bool(v) for v in ctx.test_op(43, _rows([_g2_vals(b) for b in qs]))[:, 0]] == [False] * len(qs)
    assert not any(g2_in_subgroup(b) for b in qs)


def test_small_order_b_verdicts(ctx, small_order_points):
    """verify_many agrees with the host verifier (whose affine loop meets no vertical line for these orders); verify_batch
    and both compressed verifiers, which check that B lies in G2, reject"""
    from circom_compat_b200 import Groth16, release
    from circom_compat_b200 import ethereum as eth
    vk, logs, ic, rng = _edge_key(710, 1, lambda j, r: r.randrange(1, R))
    al, be, ga, de = logs
    pvk = V.prepare_verifying_key(vk)
    inputs, proofs = [], []
    for _, b in small_order_points:
        xs = [rng.randrange(R)]
        prep = (ic[0] + xs[0] * ic[1]) % R
        c = -(al * be + prep * ga) * pow(de, -1, R) % R
        inputs += [xs, xs]
        proofs += [_proof(None, b, _g1(c)),                                          # e(A, B) drops out: host accepts
                   _proof(_g1(rng.randrange(1, R)), b, _g1(rng.randrange(1, R)))]
    assert all(_affine_walk_is_regular(b) for _, b in small_order_points)
    want = [V.verify_with_processed_vk(pvk, xs, p) for xs, p in zip(inputs, proofs)]
    assert want[0::2] == [True] * len(small_order_points)
    assert Groth16.verify_many(vk, inputs, proofs, ctx) == want
    blobs = [eth.serialize_compressed(eth.Proof.from_proof(p)) for p in proofs]
    assert Groth16.decompress_proofs(blobs, ctx) == [None] * len(blobs)
    assert Groth16.verify_many_compressed(vk, inputs, blobs, ctx) == [False] * len(blobs)
    for j in range(len(proofs)):
        assert not Groth16.verify_batch(vk, [inputs[j]], [proofs[j]], ctx)
        assert not Groth16.verify_batch_compressed(vk, [inputs[j]], [blobs[j]], ctx)
    release(vk)
