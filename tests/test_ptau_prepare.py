"""Prepared powers-of-tau ceremonies: the Lagrange sections 12-15 (ptau.read_ptau / write_ptau, b2g_powers_prepare,
b2g_lagrange_check, b2g_setup_from_lagrange; Groth16.prepare_powers_of_tau and the Lagrange routes of
generate_parameters_from_powers_of_tau and verify_powers_of_tau).  CPU: the container round trip, the check's scalar identity
and the H correction in exact integers.  GPU: every prepared block against fixed-base products of the scalar transform, keys
byte for byte against the transform route and b2g_setup, and each forgery of a Lagrange section refused with its reason."""
import ctypes as C
import io
import random

import numpy as np
import pytest

from circom_compat_b200 import Lagrange, Powers, read_ptau, synth, write_ptau
from circom_compat_b200.ptau import LAGRANGE, lagrange_counts
from circom_compat_b200.zkey import Q_MOD, R_MOD
import ptau_model as P

ARRAYS = ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'delta_g1', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')


def _rows(power, seed=1):
    rng = np.random.default_rng(seed)
    n = 1 << power
    return [rng.integers(0, 1 << 63, size=s, dtype=np.uint64) for s in ((2 * n - 1, 8), (n, 16), (n, 8), (n, 8), (1, 16))]


def _lag_rows(power, seed=2):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 1 << 63, size=(c, 16 if k == 'tau_g2' else 8), dtype=np.uint64)
            for k, c in zip(LAGRANGE, lagrange_counts(power))]


def _prepared(power, seed=1):
    return Powers(power, power + 1, *_rows(power, seed), lagrange=Lagrange(power, *_lag_rows(power, seed + 1)))


def _bytes(powers) -> bytes:
    f = io.BytesIO()
    write_ptau(f, powers)
    return f.getvalue()


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize('power', [1, 3, 6])
def test_prepared_container_round_trip(tmp_path, power):
    pw = _prepared(power, power)
    path = tmp_path / 'prep.ptau'
    write_ptau(str(path), pw)
    for src in (str(path), path.read_bytes()):
        got = read_ptau(src)
        assert (got.power, got.ceremony_power) == (power, power + 1)
        for k in ARRAYS:
            assert getattr(got, k).tobytes() == getattr(pw, k).tobytes(), k
        assert got.lagrange is not None and got.lagrange.power == power
        for k in LAGRANGE:
            assert getattr(got.lagrange, k).tobytes() == getattr(pw.lagrange, k).tobytes(), k


@pytest.mark.parametrize('power', [1, 4])
def test_unprepared_writer_output_equals_the_model(power):
    rows = _rows(power, 5)
    assert _bytes(Powers(power, power + 3, *rows)) == P.write_ptau(power, *rows, ceremony_power=power + 3)


def test_a_prefix_object_is_refused_by_the_writer():
    with pytest.raises(ValueError, match='section 2 needs'):
        _bytes(_prepared(4).prefix(2))


@pytest.mark.parametrize('case', ['missing 12', 'missing 13', 'missing 15', 'short 14', 'long 12'])
def test_incomplete_lagrange_sections_read_as_none(case):
    power = 3
    rows, lag = _rows(power, 7), _lag_rows(power, 8)
    secs = [P.header(power)] + [P.section(2 + k, r.tobytes()) for k, r in enumerate(rows)]
    body = {12 + k: a.tobytes() for k, a in enumerate(lag)}
    what, sid = case.split()
    sid = int(sid)
    if what == 'missing':
        del body[sid]
    elif what == 'short':
        body[sid] = body[sid][:-64]
    else:
        body[sid] += b'\0' * 64
    pw = read_ptau(P.container(secs + [P.section(s, b) for s, b in body.items()]))
    assert pw.lagrange is None and pw.tau_g1.tobytes() == rows[0].tobytes()


def test_prefix_carries_the_lagrange_blocks():
    """prefix(k) keeps blocks 0 .. k + 1 / 0 .. k, equal to the prepared file of power k written from the same rows, except
    for the extra tau_g1 row that the unpadded top block reads below the prepared power"""
    p = 6
    pw = read_ptau(_bytes(_prepared(p, 3)))
    for k in range(1, p + 1):
        n = 1 << k
        for copy in (False, True):
            got = pw.prefix(k, copy=copy)
            assert got.tau_g1.shape[0] == (2 * n if k < p else 2 * n - 1)
            small = Powers(k, pw.ceremony_power, got.tau_g1[:2 * n - 1], got.tau_g2, got.alpha_tau_g1, got.beta_tau_g1, got.beta_g2,
                           lagrange=Lagrange(k, *(getattr(got.lagrange, x) for x in LAGRANGE)))
            back = read_ptau(_bytes(small))
            for x, c in zip(LAGRANGE, lagrange_counts(k)):
                a = getattr(pw.lagrange, x)[:c]
                assert getattr(got.lagrange, x).tobytes() == a.tobytes() == getattr(back.lagrange, x).tobytes(), (k, x)
            assert got.lagrange.power == p
    with pytest.raises(ValueError, match='exceeds'):
        pw.prefix(p + 1)


def _weights_to_scalars(p, log_n, rho, section12):
    """s = sum_k pad(iNTT_(2^k)(w_k)) over the blocks the check reads, w at global index g = rho^g"""
    top = log_n + 1 if section12 else log_n
    s = [0] * (1 << top)
    for k in range(top + 1):
        m = 1 << k
        t = P.intt([pow(rho, m - 1 + i, R_MOD) for i in range(m)])
        for j in range(m):
            s[j] = (s[j] + t[j]) % R_MOD
    if section12 and log_n == p:
        s[-1] = 0                                  # the padding infinity's coefficient
    return s


@pytest.mark.parametrize('p,log_n', [(1, 1), (2, 1), (3, 3), (3, 2)])
def test_check_scalar_identity(p, log_n):
    """sum w . Lambda = sum s . X in exact integers, X the scalars of the monomials, Lambda the prepared blocks (tau_g1's top
    block padded at log_n = p)"""
    rng = random.Random(p * 10 + log_n)
    tau, rho = rng.randrange(1, R_MOD), rng.randrange(1, R_MOD)
    n = 1 << p
    mono = [pow(tau, i, R_MOD) for i in range(2 * n - 1)] + [0]      # tau_g1 of power p, then the padding
    for section12 in (True, False):
        top = log_n + 1 if section12 else log_n
        lam = []
        for k in range(top + 1):
            m = 1 << k
            lam += P.intt(mono[:m] if not (section12 and k == p + 1) else mono[:2 * n])
        lhs = sum(pow(rho, g, R_MOD) * v for g, v in enumerate(lam)) % R_MOD
        s = _weights_to_scalars(p, log_n, rho, section12)
        rhs = sum(a * b for a, b in zip(s, mono)) % R_MOD
        assert lhs == rhs, (p, log_n, section12)
        lam[len(lam) // 2] = (lam[len(lam) // 2] * 2) % R_MOD          # a forged entry breaks it
        assert sum(pow(rho, g, R_MOD) * v for g, v in enumerate(lam)) % R_MOD != rhs


@pytest.mark.parametrize('n', [1, 2, 4, 16])
def test_h_correction_identity(n):
    """the odd entries of iNTT_2n(tau^0 .. tau^(2n-1)) less (2n)^-1 omega_2n^(2i+1) tau^(2n-1) are the reference's H, also with
    tau in the domain"""
    w = synth.root_of_unity(2 * n)
    inv = pow(2 * n, -1, R_MOD)
    for tau in [random.Random(n).randrange(1, R_MOD)] + [pow(w, k, R_MOD) for k in (0, 1, n)]:
        full = P.intt([pow(tau, i, R_MOD) for i in range(2 * n)])
        last = pow(tau, 2 * n - 1, R_MOD)
        got = [(full[2 * i + 1] - inv * pow(w, 2 * i + 1, R_MOD) * last) % R_MOD for i in range(n)]
        assert got == P.folded_circom_h(n, tau)
        if pow(tau, 2 * n, R_MOD) != 1:
            assert got == synth.h_query_scalars(n, tau, 1)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope='module')
def gpu():
    from circom_compat_b200 import Context, release_all
    c = Context(0)
    yield c
    release_all()
    c.close()


def _limbs(vals):
    return synth._ints_to_limbs([v % R_MOD for v in vals])


class Cer:
    """a ceremony of power p for (tau, alpha, beta) on g1 = k1 G1, g2 = k2 G2 by fixed-base products, with its scalars"""

    def __init__(self, ctx, power, tau, alpha, beta, k1=1, k2=1):
        self.power, self.tau, self.alpha, self.beta, self.k1, self.k2 = power, tau, alpha, beta, k1, k2
        n = 1 << power
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * tau % R_MOD
        self.t = t
        self.powers = Powers(power, power, ctx.fixed_base_g1(_limbs([k1 * v for v in t])), ctx.fixed_base_g2(_limbs([k2 * v for v in t[:n]])),
                             ctx.fixed_base_g1(_limbs([k1 * alpha * v for v in t[:n]])),
                             ctx.fixed_base_g1(_limbs([k1 * beta * v for v in t[:n]])), ctx.fixed_base_g2(_limbs([k2 * beta])))

    def generators(self):
        return (None, None) if self.k1 == self.k2 == 1 else (self.powers.tau_g1[0], self.powers.tau_g2[0])

    def expected_blocks(self, ctx, K):
        """sections 12-15 of the ceremony of power K formed by this one's prefix: fixed-base products of iNTT_(2^k)(scalars)"""
        nK = 1 << K
        mono = {'tau_g1': [self.k1 * v for v in self.t[:2 * nK - 1]] + [0], 'tau_g2': [self.k2 * v for v in self.t[:nK]],
                'alpha_tau_g1': [self.k1 * self.alpha * v for v in self.t[:nK]],
                'beta_tau_g1': [self.k1 * self.beta * v for v in self.t[:nK]]}
        out = {}
        for name in LAGRANGE:
            top = K + 1 if name == 'tau_g1' else K
            vals = []
            for k in range(top + 1):
                vals += P.intt(mono[name][:1 << k])
            fb = ctx.fixed_base_g2 if name == 'tau_g2' else ctx.fixed_base_g1
            out[name] = fb(_limbs(vals))
        return out


_CER = {}


def _cer(ctx, power, seed=7, k1=1, k2=1, tau=None):
    key = (power, seed, k1, k2, tau)
    if key not in _CER:
        rng = random.Random(seed)
        t, a, b = (rng.randrange(1, R_MOD) for _ in range(3))
        _CER[key] = Cer(ctx, power, tau if tau is not None else t, a, b, k1, k2)
    return _CER[key]


_PREP = {}


def _prep(ctx, power, **kw):
    from circom_compat_b200 import Groth16
    key = (power, tuple(sorted(kw.items())))
    if key not in _PREP:
        _PREP[key] = Groth16.prepare_powers_of_tau(_cer(ctx, power, **kw).powers, ctx=ctx)
    return _PREP[key]


@pytest.mark.gpu
@pytest.mark.parametrize('power', list(range(1, 13)))
def test_prepare_matches_fixed_base_of_the_scalar_transform(gpu, power):
    from circom_compat_b200 import Groth16
    cers = [_cer(gpu, power)]
    if power in (3, 8):
        w = synth.root_of_unity(1 << power)
        cers += [_cer(gpu, power, tau=w), _cer(gpu, power, seed=9, k1=7, k2=5)]
    for c in cers:
        got = Groth16.prepare_powers_of_tau(c.powers, ctx=gpu)
        want = c.expected_blocks(gpu, power)
        assert got.power == power and got.lagrange.power == power
        for name in LAGRANGE:
            assert getattr(got.lagrange, name).tobytes() == want[name].tobytes(), (power, name, c.tau == c.t[1])


@pytest.mark.gpu
@pytest.mark.parametrize('K', [8, 12])
def test_prepare_at_a_reduced_power(gpu, K, tmp_path):
    """powers 8 and 12 from a power-14 ceremony: block K + 1 is padded with infinity and the result equals the prepare of the
    truncated file, written to disk and read back"""
    from circom_compat_b200 import Groth16
    big = _cer(gpu, 14)
    path = tmp_path / f'prep{K}.ptau'
    got = Groth16.prepare_powers_of_tau(big.powers, dst=str(path), power=K, ctx=gpu)
    assert got.power == K and got.lagrange.power == K
    small = Groth16.prepare_powers_of_tau(big.powers.prefix(K), power=K, ctx=gpu)
    want = big.expected_blocks(gpu, K)
    for name in LAGRANGE:
        assert getattr(got.lagrange, name).tobytes() == getattr(small.lagrange, name).tobytes() == want[name].tobytes(), name
    assert got.tau_g1.shape[0] == (2 << K) - 1
    with pytest.raises(ValueError, match='outside'):
        Groth16.prepare_powers_of_tau(big.powers, power=15, ctx=gpu)


@pytest.mark.gpu
def test_prepare_above_the_segmented_pass(gpu):
    """power 16: blocks 16 and 17 run the per-block transform, the others the segmented pass"""
    from circom_compat_b200 import Groth16
    c = _cer(gpu, 16, seed=3)
    got = Groth16.prepare_powers_of_tau(c.powers, ctx=gpu)
    n = 1 << 16
    for name, words, mono in (('tau_g1', 8, [v for v in c.t] + [0]), ('tau_g2', 16, c.t[:n])):
        lag = getattr(got.lagrange, name)
        fb = gpu.fixed_base_g2 if words == 16 else gpu.fixed_base_g1
        for k in ((15, 16, 17) if name == 'tau_g1' else (15, 16)):
            m = 1 << k
            assert lag[m - 1:2 * m - 1].tobytes() == gpu.points_intt(fb(_limbs(mono[:m])), g2=words == 16).tobytes(), (name, k)


def _reduction(flavour):
    from circom_compat_b200 import CircomReduction, LibsnarkReduction
    return LibsnarkReduction if flavour == 'libsnark' else CircomReduction


def _same_key(a, b):
    for name in KEY_FIELDS:
        x, y = np.ascontiguousarray(getattr(a, name)), np.ascontiguousarray(getattr(b, name))
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), name


def _circuit(n_vars, num_inputs, rows):
    mats = []
    for x in range(3):
        r = [k for k, row in enumerate(rows) for _ in row[x]]
        c = [col for row in rows for col, _ in row[x]]
        v = [val % R_MOD for row in rows for _, val in row[x]]
        mats.append((np.array(r, dtype=np.int64), np.array(c, dtype=np.int64), v))
    return synth.Circuit(n_vars, num_inputs, len(rows), *mats)


def _circuit_of(kind, size):
    if kind == 'chain':
        return synth.chain_circuit(size)
    if kind == 'circomlike':
        return synth.circomlike_circuit(size)[0]
    return _circuit(2, 1, [([(1, 1)], [(1, 1)], [(1, 1)])])


def _setup_both(ctx, circ, c, prepared, flavour):
    from circom_compat_b200 import Groth16
    red = _reduction(flavour)
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, prepared, ctx, red)
    _same_key(pk, Groth16.generate_parameters_from_powers_of_tau(circ, c.powers, ctx, red))
    g1, g2 = c.generators()
    _same_key(pk, Groth16.generate_parameters_with_qap(circ, c.alpha, c.beta, 1, 1, g1, g2, tau=c.tau, ctx=ctx, reduction=red))
    return pk


SIZES = [('tiny', 0)] + [('chain', 1 << k) for k in (2, 3, 5, 8, 12)] + [('chain', (1 << k) - 1) for k in (3, 9, 12)] + \
        [('circomlike', k) for k in (2, 3, 6, 10, 12)]


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
@pytest.mark.parametrize('kind,size', SIZES)
def test_setup_from_a_prepared_ceremony_matches_the_transform_route(gpu, kind, size, flavour):
    """domains 2 to 2^12 from one prepared 2^12 ceremony: log n < p for most, log n = p for the largest"""
    _setup_both(gpu, _circuit_of(kind, size), _cer(gpu, 12), _prep(gpu, 12), flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_edges_tau_in_the_domain_and_other_generators(gpu, flavour):
    for p, kw in ((3, dict(tau=synth.root_of_unity(8))), (3, dict(tau=synth.root_of_unity(16))), (4, dict(seed=9, k1=7, k2=5))):
        c, prep = _cer(gpu, p, **kw), _prep(gpu, p, **kw)
        for kind, size in (('tiny', 0), ('chain', 3), ('chain', 1 << (p - 1)), ('circomlike', p)):
            circ = _circuit_of(kind, size)
            _setup_both(gpu, circ, c, prep, flavour)


@pytest.mark.gpu
@pytest.mark.parametrize('flavour', ['circom', 'libsnark'])
def test_setup_at_2_16_and_2_18(gpu, flavour):
    _setup_both(gpu, synth.circomlike_circuit(16)[0], _cer(gpu, 16), _prep(gpu, 16), flavour)
    if flavour == 'circom':
        _setup_both(gpu, synth.chain_circuit(1 << 18), _cer(gpu, 18), _prep(gpu, 18), flavour)


@pytest.mark.gpu
def test_the_key_passes_its_check_and_proves(gpu):
    from circom_compat_b200 import Groth16, fr_to_mont
    circ = synth.chain_circuit(200)
    prep = _prep(gpu, 9)
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, prep, gpu)
    assert Groth16.verify_proving_key(circ, prep, pk, ctx=gpu)
    pk2 = Groth16.contribute(pk, x=12345, ctx=gpu)
    w = synth.chain_witness(200)
    proof = Groth16.create_proof_with_reduction_and_matrices(pk2, 3, 5, circ.matrices(), circ.num_inputs, circ.num_constraints,
                                                             fr_to_mont(w), gpu)
    assert Groth16.verify(pk2, w[1:circ.num_inputs], proof)


def _forge(prep, name, i, row):
    lag = {k: np.array(getattr(prep.lagrange, k), copy=True) for k in LAGRANGE}
    lag[name][i] = row
    return Powers(prep.power, prep.ceremony_power, *(getattr(prep, k) for k in ARRAYS), lagrange=Lagrange(prep.lagrange.power, *(lag[k] for k in LAGRANGE)))


def _forge_block(prep, name, k, fn):
    lag = {x: np.array(getattr(prep.lagrange, x), copy=True) for x in LAGRANGE}
    m = 1 << k
    lag[name][m - 1:2 * m - 1] = fn(lag[name][m - 1:2 * m - 1])
    return Powers(prep.power, prep.ceremony_power, *(getattr(prep, k) for k in ARRAYS), lagrange=Lagrange(prep.lagrange.power, *(lag[x] for x in LAGRANGE)))


def _double(ctx, row, g2):
    """2 P for one affine Montgomery row, by the MSM with scalar 2"""
    pts = np.ascontiguousarray(row).reshape(1, -1)
    s = _limbs([2])
    return (ctx.msm_g2 if g2 else ctx.msm_g1)(pts, s).reshape(-1)


def _g2_outside_subgroup():
    from batch_model import twist_point_outside_g2
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % Q_MOD for v in (x0, x1, y0, y1)]).reshape(16)


@pytest.mark.gpu
def test_honest_prepared_ceremonies_pass(gpu):
    from circom_compat_b200 import Groth16
    for p in (1, 2, 5, 12):
        prep = _prep(gpu, p)
        assert Groth16.verify_powers_of_tau(prep, ctx=gpu)
        for log_n in range(1, p + 1):
            assert Groth16.verify_powers_of_tau(prep, log_n, ctx=gpu), (p, log_n)
    w = synth.root_of_unity(16)
    assert Groth16.verify_powers_of_tau(_prep(gpu, 3, tau=w), ctx=gpu)


@pytest.mark.gpu
def test_lagrange_forgeries_are_refused_with_their_reason(gpu):
    from circom_compat_b200 import Groth16
    p = 5
    prep = _prep(gpu, p)
    n = 1 << p
    cases = []
    for name in LAGRANGE:
        g2 = name == 'tau_g2'
        top = p + 1 if name == 'tau_g1' else p
        arr = getattr(prep.lagrange, name)
        not_tf = f"lagrange_{name} is not the transform of {name}"
        for k in (0, 3, top):
            i = (1 << k) - 1 + (1 << k) // 2
            cases.append((f'{name} block {k} doubled', _forge(prep, name, i, _double(gpu, arr[i], g2)), not_tf))
        cases.append((f'{name} swapped', _forge_block(prep, name, 3, lambda b: b[[1, 0] + list(range(2, len(b)))]), not_tf))
        br = [int(format(j, '03b')[::-1], 2) for j in range(8)]
        cases.append((f'{name} bit-reversed', _forge_block(prep, name, 3, lambda b: b[br]), not_tf))
        a = np.array(arr[7:15], copy=True)
        scaled = np.stack([_double(gpu, r, g2) for r in a])                     # 2^-k scaling missed by a factor of 2
        cases.append((f'{name} unscaled', _forge_block(prep, name, 3, lambda b: scaled), not_tf))
        i = 9
        bad = np.array(arr[i], copy=True); bad[4 if not g2 else 8] ^= 1
        cases.append((f'{name} off its curve', _forge(prep, name, i, bad), f"lagrange_{name}[{i}]: off the {'twist' if g2 else 'curve'}"))
        bad = np.array(arr[i], copy=True); bad[3] = (1 << 64) - 1
        cases.append((f'{name} coordinate', _forge(prep, name, i, bad), f"lagrange_{name}[{i}]: a coordinate >= p"))
    cases.append(('tau_g2 outside G2', _forge(prep, 'tau_g2', 20, _g2_outside_subgroup()), 'lagrange_tau_g2[20]: not in G2'))
    cases.append(('top block padded with T_0', _forge_block(prep, 'tau_g1', p + 1,
                                                             lambda b: gpu.points_intt(np.concatenate([prep.tau_g1, prep.tau_g1[:1]]))),
                  "lagrange_tau_g1 is not the transform of tau_g1"))
    for name, forged, reason in cases:
        got = Groth16.verify_powers_of_tau(forged, ctx=gpu)
        assert not got and got.reason == reason, (name, got.reason)
    assert n == 32


@pytest.mark.gpu
def test_a_forged_block_above_log_n_passes_the_prefix_check(gpu):
    from circom_compat_b200 import Groth16
    prep = _prep(gpu, 6)
    forged = _forge(prep, 'alpha_tau_g1', (1 << 6) - 1 + 3, prep.lagrange.alpha_tau_g1[0])
    assert not Groth16.verify_powers_of_tau(forged, ctx=gpu)
    assert Groth16.verify_powers_of_tau(forged, 5, ctx=gpu)
    forged = _forge(prep, 'tau_g1', (1 << 7) - 1 + 3, prep.lagrange.tau_g1[0])
    assert not Groth16.verify_powers_of_tau(forged, ctx=gpu)
    assert Groth16.verify_powers_of_tau(forged, 5, ctx=gpu)


@pytest.mark.gpu
def test_fixed_rho_gives_the_models_verdict(gpu):
    """at p <= 3, a fixed rho: the big-int sums of both sides decide as the device does"""
    from circom_compat_b200 import Groth16
    for p in (1, 2, 3):
        prep = _prep(gpu, p)
        ch = [random.Random(p).randrange(1, R_MOD) for _ in range(6)]
        assert Groth16.verify_powers_of_tau(prep, ctx=gpu, challenges=ch)
        forged = _forge(prep, 'beta_tau_g1', 1, prep.lagrange.beta_tau_g1[2])
        assert not Groth16.verify_powers_of_tau(forged, ctx=gpu, challenges=ch)
        assert not Groth16.verify_powers_of_tau(forged, ctx=gpu, challenges=ch[:5] + [1])


@pytest.mark.gpu
def test_forgeries_on_both_sides_of_a_slice_boundary(gpu):
    """power 21: section 12 holds 2^23 - 1 points, so block 22 straddles the 2^22-point slice boundary"""
    from circom_compat_b200 import Groth16
    p = 21
    prep = _prep(gpu, p)
    SLICE = 1 << 22
    for i in (SLICE - 1, SLICE):
        forged = _forge(prep, 'tau_g1', i, prep.lagrange.tau_g1[i - 5])
        got = Groth16.verify_powers_of_tau(forged, ctx=gpu)
        assert not got and got.reason == "lagrange_tau_g1 is not the transform of tau_g1", i
        bad = np.array(prep.lagrange.tau_g1[i], copy=True); bad[4] ^= 1
        got = Groth16.verify_powers_of_tau(_forge(prep, 'tau_g1', i, bad), ctx=gpu)
        assert got.reason == f"lagrange_tau_g1[{i}]: off the curve", i
    assert Groth16.verify_powers_of_tau(prep, ctx=gpu)


@pytest.mark.gpu
def test_errors_leave_the_context_usable(gpu):
    from circom_compat_b200 import Groth16, _native as N, fr_to_mont
    prep = _prep(gpu, 5)

    def still_usable():
        assert Groth16.verify_powers_of_tau(prep, ctx=gpu)

    pd, keep = N.PowersDesc(), []
    pd.log_size = 5
    for k in ARRAYS:
        a = np.ascontiguousarray(getattr(prep, k)); keep.append(a); setattr(pd, k, a.ctypes.data)
    ld = N.LagrangeDesc()
    ld.log_size = 5
    for k in LAGRANGE:
        a = np.ascontiguousarray(getattr(prep.lagrange, k)); keep.append(a); setattr(ld, k, a.ctypes.data)
    rho = np.frombuffer((3).to_bytes(32, 'little'), dtype=np.uint8).copy()
    rep = N.PowersReport()
    L = N.lib()
    assert L.b2g_lagrange_check(gpu._h, C.byref(pd), C.byref(ld), 5, rho.ctypes.data, C.byref(rep)) == N.B2G_OK and rep.ok
    still_usable()
    assert L.b2g_lagrange_check(gpu._h, C.byref(pd), C.byref(ld), 6, rho.ctypes.data, C.byref(rep)) == N.B2G_E_DOMAIN
    assert L.b2g_lagrange_check(gpu._h, C.byref(pd), C.byref(ld), 0, rho.ctypes.data, C.byref(rep)) == N.B2G_E_DOMAIN
    zero = np.zeros(32, dtype=np.uint8)
    assert L.b2g_lagrange_check(gpu._h, C.byref(pd), C.byref(ld), 5, zero.ctypes.data, C.byref(rep)) == N.B2G_E_INPUT
    assert L.b2g_lagrange_check(gpu._h, C.byref(pd), None, 5, rho.ctypes.data, C.byref(rep)) == N.B2G_E_SHAPE
    still_usable()
    out = N.LagrangeDesc()
    out.log_size = 6
    assert L.b2g_powers_prepare(gpu._h, C.byref(pd), C.byref(out)) == N.B2G_E_DOMAIN
    out.log_size = 5
    assert L.b2g_powers_prepare(gpu._h, C.byref(pd), C.byref(out)) == N.B2G_E_SHAPE
    bad = np.array(prep.tau_g2, copy=True); bad[17] = _g2_outside_subgroup()
    with pytest.raises(N.B2gError, match=r'tau_g2\[17\]: not in G2'):
        Groth16.prepare_powers_of_tau(Powers(5, 5, prep.tau_g1, bad, prep.alpha_tau_g1, prep.beta_tau_g1, prep.beta_g2), ctx=gpu)
    still_usable()
    circ = synth.chain_circuit(20)
    bad = np.array(prep.lagrange.tau_g2, copy=True); bad[40] = _g2_outside_subgroup()
    forged = Powers(5, 5, *(getattr(prep, k) for k in ARRAYS), lagrange=Lagrange(5, prep.lagrange.tau_g1, bad,
                                                                                 prep.lagrange.alpha_tau_g1, prep.lagrange.beta_tau_g1))
    with pytest.raises(N.B2gError, match=r'lagrange_tau_g2\[40\]: not in G2'):
        Groth16.generate_parameters_from_powers_of_tau(circ, forged, gpu)
    with pytest.raises(N.PolynomialDegreeTooLarge):
        Groth16.generate_parameters_from_powers_of_tau(synth.chain_circuit(100), prep, gpu)
    still_usable()
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, prep, gpu)
    w = synth.chain_witness(20)
    pending = Groth16.submit(pk, 5, 7, circ.matrices(), fr_to_mont(w), gpu)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.verify_powers_of_tau(prep, ctx=gpu)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.prepare_powers_of_tau(prep, ctx=gpu)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.generate_parameters_from_powers_of_tau(circ, prep, gpu)
    assert Groth16.verify(pk, w[1:circ.num_inputs], pending.wait())
    still_usable()


@pytest.mark.gpu
def test_cpp_prepare_and_setup_modes_match_python(gpu, tmp_path):
    """B2G_PTAU_PREPARE=<in.ptau> groth16_bench <out.ptau> [power] writes the file Python writes, and B2G_SETUP_PTAU on the
    prepared file makes the key it makes on the unprepared one"""
    import os
    import subprocess
    from circom_compat_b200 import Groth16
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    golden = os.path.join(root, 'tests', 'golden')
    exe = os.path.join(root, 'circom_compat_b200', 'host', 'groth16_bench')
    c = _cer(gpu, 9, seed=21)
    src = tmp_path / 'pot9.ptau'
    write_ptau(str(src), c.powers)
    for power in (None, 8):
        out = tmp_path / f'prep{power}.ptau'
        args = [exe, str(out)] + ([str(power)] if power else [])
        subprocess.check_output(args, text=True, env=dict(os.environ, B2G_PTAU_PREPARE=str(src)))
        py = tmp_path / f'py{power}.ptau'
        Groth16.prepare_powers_of_tau(c.powers, dst=str(py), power=power, ctx=gpu)
        assert out.read_bytes() == py.read_bytes(), power
    keys = []
    for path in (src, tmp_path / 'prepNone.ptau'):
        res = subprocess.check_output([exe, os.path.join(golden, 'circuit2.r1cs'), os.path.join(golden, 'circuit2_witness.wtns'), '0x77'],
                                      text=True, env=dict(os.environ, B2G_SETUP_PTAU=str(path)))
        kv = dict(line.split('=', 1) for line in res.splitlines() if '=' in line)
        assert kv['contribution'] == '1' and kv['verified'] == '1'
        keys.append(kv['key'])
    assert keys[0] == keys[1]
