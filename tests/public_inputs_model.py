"""Circuits with many public inputs, and the CPU references tests/test_public_inputs.py holds the device against.
TEST INFRASTRUCTURE ONLY.

public_circuit builds an R1CS whose public inputs take any values: each constraint's C target is a fresh private wire
computed forward from A.w * B.w over earlier wires, so the witness of any public-input values satisfies the circuit.  The
modes place the public inputs in the matrices (only in their input rows, in A, B or C rows with coefficients 1, r - 1 and
random, one input in every row, or every wire public so that L is empty).  SHAPES picks (m, num_inputs) pairs that cross
the boundaries two public inputs never reach: one 256-thread CTA of input rows, input rows that fill or decide the domain,
an empty IC tail (n_public = 0), an empty L query, and 2049 inputs.

The references: the proof dlogs of a trapdoor key without any h (both reductions, satisfying witnesses), the key-check
equations E1-E5 for given key scalars (so that a forged key's broken equation is predicted), and the count rule."""
import random

import numpy as np

from circom_compat_b200 import synth
from circom_compat_b200.zkey import R_MOD
import setup_check_model as SC

R = R_MOD
MODES = ('unused', 'in_a', 'in_b', 'in_c', 'hot', 'all_public')

# name: (m, num_inputs (w0 and the public inputs), n_vars, mode)
SHAPES = {
    'p0': (1, 1, 4, 'unused'),               # n_public = 0: IC holds w0 alone
    'p254': (5, 255, 300, 'in_a'),           # 255 input rows: one short of a 256-thread CTA
    'p255': (5, 256, 300, 'in_b'),           # exactly one CTA of input rows
    'p256': (5, 257, 300, 'in_c'),           # one input row past it
    'fill1024': (1, 1023, 1030, 'hot'),      # m + num_inputs = 1024: the input rows fill the domain
    'over1024': (1, 1024, 1030, 'in_a'),     # m + num_inputs = 1025: the input rows decide the domain of 2048
    'ordinary': (2000, 48, 2100, 'in_c'),    # an ordinary circuit, m + num_inputs = 2048
    'wide': (3000, 1100, 8192, 'hot'),       # n_vars 8192, domain 8192
    'most': (100, 2049, 2200, 'in_a'),       # the largest input count
    'all_public': (40, 300, 300, 'all_public'),
}


def _coef(k, rng):
    return (1, R - 1, rng.randrange(2, R - 1))[k % 3]


def public_circuit(m, num_inputs, n_vars, mode, seed=0):
    """(synth.Circuit, witness) where witness(publics, seed) is the full assignment [1, *publics, private wires] that satisfies
    the circuit for any list of num_inputs - 1 public values"""
    assert mode in MODES
    ni = num_inputs
    rng = random.Random(seed * 7919 + m * 31 + ni)
    rows = [([], [], []) for _ in range(m)]                  # per row: A, B, C lists of (column, coefficient)
    pubs = list(range(1, ni))
    if mode == 'all_public':
        assert n_vars == ni and ni > 1
        for k in range(m):                                    # c * w_j (+ d * w_j2) times w0 = the same: true for any w
            terms = [(pubs[k % len(pubs)], _coef(k, rng))]
            if k % 4 == 1:
                terms.append((pubs[(k * 37 + 11) % len(pubs)], _coef(k + 1, rng)))
            rows[k] = (terms, [(0, 1)], list(terms))
        outs, free = [], []
    else:
        priv = n_vars - ni
        assert priv >= m, (m, ni, n_vars)
        free = list(range(ni, ni + priv - m))                 # private wires the witness draws
        outs = list(range(ni + priv - m, n_vars))             # row k's C target
        for k in range(m):
            src = [0] + free + outs[:k]
            rows[k][0].append((rng.choice(src), _coef(k, rng)))
            if k % 3 == 2:
                rows[k][0].append((rng.choice(src), _coef(k + 1, rng)))
            rows[k][1].append((rng.choice(src), _coef(k + 2, rng)))
            rows[k][2].append((outs[k], _coef(k, rng) if k % 5 else 1))
        if mode in ('in_a', 'in_b', 'in_c'):
            x = 'abc'.index(mode[-1])
            for j in pubs:                                    # every input in one or two rows, coefficients 1, r - 1, random
                for k in sorted({(j - 1) % m, (7 * j + 3) % m}):
                    rows[k][x].append((j, _coef(j + k, rng)))
        elif mode == 'hot' and pubs:
            hot = pubs[-1]
            for k in range(m):
                for x in range(3):
                    rows[k][x].append((hot, _coef(k + x, rng)))
    mats = []
    for x in range(3):
        r = [k for k in range(m) for _ in rows[k][x]]
        c = [col for k in range(m) for col, _ in rows[k][x]]
        v = [val for k in range(m) for _, val in rows[k][x]]
        mats.append((np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), v))
    circ = synth.Circuit(n_vars, ni, m, *mats)

    def witness(publics, wseed=1):
        publics = [int(v) % R for v in publics]
        assert len(publics) == ni - 1
        wr = random.Random(wseed)
        w = [1] + publics + [0] * (n_vars - ni)
        for i in free:
            w[i] = wr.randrange(R) if i % 3 else wr.randrange(2)
        for k in range(m):
            a = sum(v * w[col] for col, v in rows[k][0]) % R
            b = sum(v * w[col] for col, v in rows[k][1]) % R
            if outs:
                (out, cv), rest = rows[k][2][0], rows[k][2][1:]
                w[out] = (a * b - sum(v * w[col] for col, v in rest)) * pow(cv, -1, R) % R
        return w

    return circ, witness


def shape_circuit(name, seed=0):
    return public_circuit(*SHAPES[name], seed=seed)


def public_values(num_public, seed=5):
    """the public-input vectors the tests prove: all 0, all 1, all r - 1, and random ones"""
    rng = random.Random(seed)
    return [[0] * num_public, [1] * num_public, [R - 1] * num_public, [rng.randrange(R) for _ in range(num_public)]]


def unsatisfied_rows(circ, w):
    """the rows k where (A_k . w)(B_k . w) != C_k . w"""
    ev = []
    for rows, cols, vals in (circ.A, circ.B, circ.C):
        e = [0] * circ.num_constraints
        for r, c, v in zip(np.asarray(rows).tolist(), np.asarray(cols).tolist(), vals):
            e[r] = (e[r] + v * w[c]) % R
        ev.append(e)
    return [k for k in range(circ.num_constraints) if ev[0][k] * ev[1][k] % R != ev[2][k]]


def proof_dlogs(td, circ, w, r, s):
    """dlog(A), dlog(B), dlog(C) of the proof of a satisfying assignment under a trapdoor key of either flavour, with the H
    term (a(tau) b(tau) - c(tau)) / delta: for a satisfying assignment the LibsnarkReduction h is the exact quotient by Z, so
    sum_j h_j tau^j Z(tau) / delta is that same term, as it is for every assignment under CircomReduction"""
    assert not unsatisfied_rows(circ, w)
    saved = td.flavour
    td.flavour = 'circom'
    try:
        return synth.expected_proof_dlogs_independent(td, circ, w, r, s)
    finally:
        td.flavour = saved


# ------------------------------------------------------------------------------------------------ the key check
EQUATION_REASONS = {'a_query': 'a_query does not match the circuit and ceremony',
                    'b_g1_query': 'b_g1_query does not match the circuit and ceremony',
                    'b_g2_query': 'b_g2_query does not match the circuit and ceremony',
                    'gamma_abc_g1 / l_query': 'gamma_abc_g1 / l_query do not match the circuit and ceremony',
                    'h_query': 'h_query does not match the circuit and ceremony'}


def key_equations(circ, key, tau, alpha, beta, delta, rho, sigma, flavour):
    """E1-E5 in the exponent for the key scalars `key` (setup_check_model.key_scalars' dict, possibly edited): a list of
    (name, key side, ceremony side), in the order b2g_setup_check reports them"""
    w, v, sa, sb, sc, h = SC.scalars(circ, rho, sigma, flavour)
    ni = circ.num_inputs

    def at_tau(s, scale=1):
        acc, p = 0, 1
        for x in s:
            acc += x * p
            p = p * tau % R
        return acc * scale % R

    def weighted(vals, start=0):
        return sum(w[start + j] * x for j, x in enumerate(vals)) % R

    assert len(key['ic']) == ni and len(key['l']) == circ.n_vars - ni
    e4_key = (weighted(key['ic']) + delta * weighted(key['l'], ni)) % R
    e4_cer = (at_tau(sa, beta) + at_tau(sb, alpha) + at_tau(sc)) % R
    e5_key = delta * sum(x * y for x, y in zip(v, key['h'])) % R
    return [('a_query', weighted(key['a']), at_tau(sa)), ('b_g1_query', weighted(key['b']), at_tau(sb)),
            ('b_g2_query', weighted(key['b']), at_tau(sb)), ('gamma_abc_g1 / l_query', e4_key, e4_cer), ('h_query', e5_key, at_tau(h))]


def broken_equations(circ, key, tau, alpha, beta, delta, rho, sigma, flavour):
    return [name for name, k, c in key_equations(circ, key, tau, alpha, beta, delta, rho, sigma, flavour) if k != c]


# key-scalar forgeries: (name, edit of the scalar dict).  IC[n_public] <-> L[0] swaps the two points either side of the rho
# offset ni; the others add the generator to one point
def _swap_ic_l(k):
    k['ic'][-1], k['l'][0] = k['l'][0], k['ic'][-1]


def _bump(field, index):
    def edit(k):
        k[field][index] = (k[field][index] + 1) % R
    return edit


def forgeries(ni, n_l):
    """[(name, edit)] of the forgeries a key with ni IC points and n_l L points admits"""
    out = [('IC[middle] + G', _bump('ic', ni // 2))]
    if n_l:
        out = [('IC[n_public] <-> L[0]', _swap_ic_l)] + out + [('L[0] + G', _bump('l', 0))]
    return out


def edited(key, edit):
    k = {name: list(v) for name, v in key.items()}
    edit(k)
    return k


def count_rule(circ, n_vars, n_ic, n_l, n_h, flavour):
    """(field, index) of b2g_setup_check's count rule 6 for a key of these counts, None when they are the circuit's: the
    first of a_query, gamma_abc_g1, l_query, h_query whose count differs, with the count the circuit needs"""
    n = circ.domain_size
    for field, have, want in (('a_query', n_vars, circ.n_vars), ('gamma_abc_g1', n_ic, circ.num_inputs),
                              ('l_query', n_l, circ.n_vars - circ.num_inputs), ('h_query', n_h, n - (flavour == 'libsnark'))):
        if have != want:
            return field, want
    return None


def b_compaction(pk, lo, hi):
    """b2g_pk_load's per-shard B compaction: the number of real B points a rank keeps over its slice [lo, hi) of w[1..], or
    None when the rank does not compact (fewer than 1024 bases, or 80 % or more of them real)"""
    b1 = np.asarray(pk.b_g1_query).reshape(pk.n_vars, -1)[1 + lo:1 + hi]
    b2 = np.asarray(pk.b_g2_query).reshape(pk.n_vars, -1)[1 + lo:1 + hi]
    real = int(np.count_nonzero(b1.any(axis=1) | b2.any(axis=1)))
    return real if hi - lo >= 1024 and real * 5 < (hi - lo) * 4 else None
