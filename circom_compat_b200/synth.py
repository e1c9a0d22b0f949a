"""Synthetic circuits and trapdoor-known Groth16 setups (snarkjs flavour) for benchmarks and large parity tests.

The reference's bench family is the squaring chain (test-vectors/complex-circuit/complex-circuit.circom.template);
its only committed key has 10 000 constraints, and neither snarkjs nor a Rust toolchain exists here to make bigger
ones.  This module manufactures them: matrices + witness on the host, and a proving key whose every base is
[k]G for a scalar k derived from a known trapdoor (tau, alpha, beta, delta; gamma = 1), with the group elements computed
on the GPU by b2g_fixed_base_g1/g2.  Semantics follow generate_random_parameters_with_reduction as ark-circom uses it
(tests/groth16.rs:25) with CircomReduction::h_query_scalars (/root/reference/src/circom/qap.rs:90-105) for H, and the
public-input rows appended to A as snarkjs does (zkey section 4, src/zkey.rs:171-175).  Because the trapdoor is known,
the expected proof for any (witness, r, s) is a closed-form discrete log (tests use that as an independent check).
"""
from __future__ import annotations

import hashlib
import random
import struct
from dataclasses import dataclass

import numpy as np

from .zkey import ConstraintMatrices, ProvingKey, R_MOD, csr_from_coo

_MONT_R = 1 << 256
_ROOT_2_28 = pow(5, (R_MOD - 1) >> 28, R_MOD)


def _ints_to_limbs(vals) -> np.ndarray:
    buf = b''.join(int(v).to_bytes(32, 'little') for v in vals)
    return np.frombuffer(buf, dtype='<u8').reshape(-1, 4).copy() if buf else np.zeros((0, 4), dtype=np.uint64)


def _to_mont_limbs(vals) -> np.ndarray:
    return _ints_to_limbs([(v * _MONT_R) % R_MOD for v in vals])


def _batch_inverse(vals):
    n = len(vals)
    pre = [1] * n
    acc = 1
    for i, v in enumerate(vals):
        pre[i] = acc
        acc = acc * v % R_MOD
    inv = pow(acc, -1, R_MOD)
    out = [0] * n
    for i in range(n - 1, -1, -1):
        out[i] = inv * pre[i] % R_MOD
        inv = inv * vals[i] % R_MOD
    return out


def root_of_unity(n: int) -> int:
    return pow(_ROOT_2_28, (1 << 28) // n, R_MOD)


def sha_stream_fr(seed: int, count: int, tag: bytes = b'b2g'):
    out, ctr = [], 0
    while len(out) < count:
        d = hashlib.sha256(tag + struct.pack('<QQ', seed, ctr)).digest()
        ctr += 1
        v = int.from_bytes(d, 'little') % R_MOD
        if v:
            out.append(v)
    return out


@dataclass
class Circuit:
    """R1CS as coordinate lists (row, col, value) per matrix plus sizes; values are plain ints mod r."""
    n_vars: int
    num_inputs: int            # 1 + public
    num_constraints: int
    A: tuple                   # (rows, cols, vals) numpy int64/int64/object
    B: tuple
    C: tuple

    @property
    def domain_size(self) -> int:
        n = 1
        while n < self.num_constraints + self.num_inputs:
            n <<= 1
        return n

    def matrices(self, with_c: bool = False) -> ConstraintMatrices:
        """ConstraintMatrices as read_zkey returns them (a, b only; src/zkey.rs:181-193), or with c as
        ConstraintSystem::to_matrices() does on the R1CS route (with_c, needed by LibsnarkReduction)."""
        m = self.num_constraints
        mats = []
        for rows, cols, vals in (self.A, self.B, self.C)[:3 if with_c else 2]:
            mats.append(csr_from_coo(np.asarray(rows, dtype=np.int64), np.asarray(cols, dtype=np.uint32), _to_mont_limbs(vals), m))
        cm = ConstraintMatrices(self.num_inputs, self.n_vars - self.num_inputs, m, len(mats[0][1]), len(mats[1][1]), 0, mats[0], mats[1])
        if with_c:
            cm.c = mats[2]; cm.c_num_non_zero = len(mats[2][1])
        return cm


def chain_circuit(n_vars: int) -> Circuit:
    """Squaring chain with m = n_vars - 2 constraints: (-w[k+2]) * w[k+2] = -w[k+3], the last one targets wire 1
    (decoded from complex-circuit-10000-10000.r1cs).  n_vars = 2^k gives a domain of exactly 2^k."""
    m = n_vars - 2
    rows = np.arange(m, dtype=np.int64)
    cols = rows + 2
    ccols = np.where(rows + 3 < n_vars, rows + 3, 1)
    neg1 = [R_MOD - 1] * m
    return Circuit(n_vars, 2, m, (rows, cols, neg1), (rows, cols, [1] * m), (rows, ccols, neg1))


def chain_witness(n_vars: int, a: int = 3):
    w = [0] * n_vars
    w[0] = 1
    w[2] = a % R_MOD
    for k in range(3, n_vars):
        w[k] = w[k - 1] * w[k - 1] % R_MOD
    w[1] = w[n_vars - 1] * w[n_vars - 1] % R_MOD
    return w


def circomlike_circuit(log_n: int, seed: int = 0xC1C0):
    """A product circuit whose witness has the skew of real circom circuits: ~60 % of the wires are bits, ~20 % are
    small (< 2^32) and ~20 % are full-size field elements.  Returns (Circuit, witness).  Domain = 2^log_n."""
    rng = random.Random(seed)
    n = 1 << log_n
    num_inputs = 2
    m = n - num_inputs
    pool = 256
    # wires: [1, pub, bits.., small.., wide.., products..]
    w = [1, 0]
    bits = list(range(len(w), len(w) + pool)); w += [rng.randrange(2) for _ in range(pool)]
    small = list(range(len(w), len(w) + pool)); w += [rng.randrange(1 << 16) for _ in range(pool)]
    wide = list(range(len(w), len(w) + pool)); w += [rng.randrange(R_MOD) for _ in range(pool)]
    ar, ac, av, br, bc, bv, cr, cc, cv = [], [], [], [], [], [], [], [], []
    for k in range(m):
        u = rng.random()
        src = bits if u < 0.6 else (small if u < 0.8 else wide)
        i, j = rng.choice(src), rng.choice(src)
        out = len(w)
        w.append(w[i] * w[j] % R_MOD)
        if u >= 0.6 and u < 0.8:
            pass                                         # product of two 16-bit values stays < 2^32
        ar.append(k); ac.append(i); av.append(1)
        br.append(k); bc.append(j); bv.append(1)
        cr.append(k); cc.append(out); cv.append(1)
        if k % 97 == 0:                                  # a few two-term rows with non-unit coefficients
            ar.append(k); ac.append(0); av.append(0)
    w[1] = w[-1]
    # make wire 1 (public output) consistent: add it as an alias of the last product via the last constraint's C
    cc[-1] = 1
    w.pop()
    n_vars = len(w)
    A = (np.array(ar), np.array(ac), av); B = (np.array(br), np.array(bc), bv); Cm = (np.array(cr), np.array(cc), cv)
    return Circuit(n_vars, num_inputs, m, A, B, Cm), w


def lagrange_at(n: int, tau: int):
    """L_i(tau), i < n, over the radix-2 domain of size n."""
    w = root_of_unity(n)
    zt = (pow(tau, n, R_MOD) - 1) * pow(n, -1, R_MOD) % R_MOD
    pw = [1] * n
    for i in range(1, n):
        pw[i] = pw[i - 1] * w % R_MOD
    inv = _batch_inverse([(tau - x) % R_MOD for x in pw])
    return [zt * pw[i] % R_MOD * inv[i] % R_MOD for i in range(n)]


def h_query_scalars(n: int, tau: int, delta_inv: int):
    """Closed form of CircomReduction::h_query_scalars (qap.rs:90-105) for max_power = n - 1:
    odd-index entries of iFFT_{2n}(delta^-1 tau^i, i < 2n-1):
    lambda_j = delta^-1/(2n) * (tau^(2n-1) w^j - 1) / (tau w^-j - 1),  w = omega_{2n},  j = 2k+1."""
    w = root_of_unity(2 * n)
    winv = pow(w, -1, R_MOD)
    t_top = pow(tau, 2 * n - 1, R_MOD)
    c = delta_inv * pow(2 * n, -1, R_MOD) % R_MOD
    wj, wnj = w, winv
    w2, wn2 = w * w % R_MOD, winv * winv % R_MOD
    num, den = [], []
    for _ in range(n):
        num.append((t_top * wj - 1) % R_MOD)
        den.append((tau * wnj - 1) % R_MOD)
        wj = wj * w2 % R_MOD
        wnj = wnj * wn2 % R_MOD
    inv = _batch_inverse(den)
    return [c * a % R_MOD * b % R_MOD for a, b in zip(num, inv)]


@dataclass
class Trapdoor:
    tau: int
    alpha: int
    beta: int
    delta: int
    a_t: list
    b_t: list
    l_t: list
    h_t: list
    ic_t: list


def h_query_scalars_libsnark(n: int, tau: int, delta_inv: int):
    """LibsnarkReduction::h_query_scalars (ark-groth16 0.5.0): tau^i * Z(tau) / delta for i < n - 1"""
    zt = (pow(tau, n, R_MOD) - 1) * delta_inv % R_MOD
    out, p = [], 1
    for _ in range(n - 1):
        out.append(p * zt % R_MOD)
        p = p * tau % R_MOD
    return out


def setup_scalars(circ: Circuit, seed: int = 0xB200, trapdoor=None, flavour: str = 'circom') -> Trapdoor:
    """trapdoor = (tau, alpha, beta, gamma, delta) or None (derived from `seed`, gamma = 1)"""
    if trapdoor is None:
        tau, alpha, beta, delta = sha_stream_fr(seed, 4, b'b2g-trapdoor')
        gamma = 1
    else:
        tau, alpha, beta, gamma, delta = (int(x) % R_MOD for x in trapdoor)
    n, m, li = circ.domain_size, circ.num_constraints, circ.num_inputs
    L = lagrange_at(n, tau)
    a_t = [0] * circ.n_vars; b_t = [0] * circ.n_vars; c_t = [0] * circ.n_vars
    for (rows, cols, vals), tgt in ((circ.A, a_t), (circ.B, b_t), (circ.C, c_t)):
        for r, c, v in zip(rows.tolist() if hasattr(rows, 'tolist') else rows, cols.tolist() if hasattr(cols, 'tolist') else cols, vals):
            if v:
                tgt[c] = (tgt[c] + v * L[r]) % R_MOD
    for j in range(li):                                   # public-input rows of A (qap.rs:46-50 / zkey section 4)
        a_t[j] = (a_t[j] + L[m + j]) % R_MOD
    dinv = pow(delta, -1, R_MOD)
    abc = [(beta * a_t[i] + alpha * b_t[i] + c_t[i]) % R_MOD for i in range(circ.n_vars)]
    l_t = [x * dinv % R_MOD for x in abc[li:]]
    ginv = pow(gamma, -1, R_MOD)
    h_t = h_query_scalars(n, tau, dinv) if flavour == 'circom' else h_query_scalars_libsnark(n, tau, dinv)
    td = Trapdoor(tau, alpha, beta, delta, a_t, b_t, l_t, h_t, [x * ginv % R_MOD for x in abc[:li]])
    td.gamma = gamma
    td.lagrange = L                     # L_row(tau), row < n: lets the expected proof be computed without any h (see below)
    td.flavour = flavour
    return td


def setup(ctx, circ: Circuit, seed: int = 0xB200, trapdoor=None, flavour: str = 'circom'):
    """Returns (ProvingKey, Trapdoor); all group elements are produced on the GPU (b2g_fixed_base_*).
    flavour 'circom' = snarkjs keys (CircomReduction H query), 'libsnark' = arkworks keys (domain - 1 H bases)."""
    td = setup_scalars(circ, seed, trapdoor, flavour)
    nv = circ.n_vars
    g1_scalars = [td.alpha, td.beta, td.delta] + td.ic_t + td.a_t + td.b_t + td.l_t + td.h_t
    g1 = ctx.fixed_base_g1(_ints_to_limbs(g1_scalars))
    g2 = ctx.fixed_base_g2(_ints_to_limbs([td.beta, getattr(td, 'gamma', 1), td.delta] + td.b_t))
    o = 3
    ic = g1[o:o + circ.num_inputs]; o += circ.num_inputs
    a_q = g1[o:o + nv]; o += nv
    b1_q = g1[o:o + nv]; o += nv
    l_q = g1[o:o + nv - circ.num_inputs]; o += nv - circ.num_inputs
    h_q = g1[o:o + len(td.h_t)]
    pk = ProvingKey(nv, circ.num_inputs - 1, len(td.h_t), g1[0:1], g1[1:2], g2[0:1], g2[1:2], g1[2:3], g2[2:3],
                    ic, a_q, b1_q, g2[3:3 + nv], l_q, h_q)
    return pk, td


def qap_numerator_at_tau(td: Trapdoor, circ: Circuit, w):
    """(a*b - c)(tau) computed WITHOUT any transform and without the C matrix: a, b are the interpolants of the row
    evaluations <A_row, w>, <B_row, w> (plus the public-input rows of A, qap.rs:46-50) and c interpolates their
    pointwise product (qap.rs:52-58), so a(tau) = sum_row a_row L_row(tau) etc.  O(nnz) big-int work.  This is the
    quantity sum_j h_j * h_t[j] * delta must equal; it never touches the witness map under test."""
    m, li, L = circ.num_constraints, circ.num_inputs, td.lagrange
    ra = [0] * m
    rb = [0] * m
    for (rows, cols, vals), tgt in ((circ.A, ra), (circ.B, rb)):
        for r_, c_, v in zip(np.asarray(rows).tolist(), np.asarray(cols).tolist(), vals):
            if v:
                tgt[r_] = (tgt[r_] + v * w[c_]) % R_MOD
    at = bt = ct = 0
    for i in range(m):
        li_ = L[i]
        at += ra[i] * li_
        bt += rb[i] * li_
        ct += (ra[i] * rb[i] % R_MOD) * li_
    for j in range(li):
        at += w[j] * L[m + j]
    return (at % R_MOD) * (bt % R_MOD) % R_MOD - ct % R_MOD


def expected_proof_dlogs_independent(td: Trapdoor, circ: Circuit, w, r: int, s: int):
    """dlog(A), dlog(B), dlog(C) of the unique proof for (w, r, s), with the H term taken from the trapdoor as
    (a(tau) b(tau) - c(tau)) / delta instead of from a computed h: independent of every NTT / witness-map code path
    (CircomReduction keys only: sum_j h_j H_j = [(ab - c)(tau) / delta] G1, SURVEY.md App. C.2)."""
    assert getattr(td, 'flavour', 'circom') == 'circom'
    li = circ.num_inputs
    da = (td.alpha + sum(x * y for x, y in zip(w, td.a_t)) + r * td.delta) % R_MOD
    db = (td.beta + sum(x * y for x, y in zip(w, td.b_t)) + s * td.delta) % R_MOD
    hterm = qap_numerator_at_tau(td, circ, w) * pow(td.delta, -1, R_MOD) % R_MOD
    dc = (sum(x * y for x, y in zip(w[li:], td.l_t)) + hterm + s * da + r * db - r * s % R_MOD * td.delta) % R_MOD
    return da, db, dc


def expected_proof_dlogs(td: Trapdoor, w, h, r: int, s: int, num_inputs: int):
    """dlog(A), dlog(B), dlog(C) of the unique proof for (w, h, r, s) under this trapdoor.  NOTE: takes h as an input,
    so it checks the MSMs and the assembly but NOT the witness map that produced h; expected_proof_dlogs_independent
    is the check that does."""
    da = (td.alpha + sum(x * y for x, y in zip(w, td.a_t)) + r * td.delta) % R_MOD
    db = (td.beta + sum(x * y for x, y in zip(w, td.b_t)) + s * td.delta) % R_MOD
    dc = (sum(x * y for x, y in zip(w[num_inputs:], td.l_t)) + sum(x * y for x, y in zip(h, td.h_t))
          + s * da + r * db - r * s % R_MOD * td.delta) % R_MOD
    return da, db, dc


def write_zkey(path, pk: ProvingKey, circ: Circuit):
    """Serialise as a snarkjs .zkey (layout: src/zkey.rs:1-27 doc, 73-101, 282-318; coefficients = v*R^2)."""
    from .zkey import Q_MOD
    secs = {}
    secs[1] = struct.pack('<I', 1)
    hdr = struct.pack('<I', 32) + Q_MOD.to_bytes(32, 'little') + struct.pack('<I', 32) + R_MOD.to_bytes(32, 'little')
    hdr += struct.pack('<III', pk.n_vars, pk.n_public, pk.domain_size)
    for arr in (pk.alpha_g1, pk.beta_g1, pk.beta_g2, pk.gamma_g2, pk.delta_g1, pk.delta_g2):
        hdr += np.ascontiguousarray(arr, dtype='<u8').tobytes()
    secs[2] = hdr
    secs[3] = np.ascontiguousarray(pk.gamma_abc_g1, dtype='<u8').tobytes()
    recs = []
    rr = _MONT_R * _MONT_R % R_MOD
    for mi, (rows, cols, vals) in enumerate((circ.A, circ.B)):
        for r, c, v in zip(np.asarray(rows).tolist(), np.asarray(cols).tolist(), vals):
            recs.append(struct.pack('<III', mi, r, c) + (v * rr % R_MOD).to_bytes(32, 'little'))
    for j in range(circ.num_inputs):
        recs.append(struct.pack('<III', 0, circ.num_constraints + j, j) + (rr % R_MOD).to_bytes(32, 'little'))
    secs[4] = struct.pack('<I', len(recs)) + b''.join(recs)
    secs[5] = np.ascontiguousarray(pk.a_query, dtype='<u8').tobytes()
    secs[6] = np.ascontiguousarray(pk.b_g1_query, dtype='<u8').tobytes()
    secs[7] = np.ascontiguousarray(pk.b_g2_query, dtype='<u8').tobytes()
    secs[8] = np.ascontiguousarray(pk.l_query, dtype='<u8').tobytes()
    secs[9] = np.ascontiguousarray(pk.h_query, dtype='<u8').tobytes()
    secs[10] = struct.pack('<I', 0) + bytes(64)
    with open(path, 'wb') as f:
        f.write(b'zkey' + struct.pack('<II', 1, len(secs)))
        for sid in (1, 2, 4, 3, 9, 8, 5, 6, 7, 10):
            f.write(struct.pack('<IQ', sid, len(secs[sid])) + secs[sid])
