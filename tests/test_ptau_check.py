"""The ceremony check (b2g_powers_check, Groth16.verify_powers_of_tau) and its tableless streamed MSM (b2g_powers_msm).
CPU: the big-int model of tests/ptau_check_model.py on honest and forged ceremonies, the shifted-sum identities, and the Python
entry's refusals.  GPU: b2g_powers_msm against b2g_msm_g1 / g2 with the explicit scalars rho^i; honest ceremonies from power 1
to 22 (at 22, tau_g1 spans two slices of 2^22 points); every kind of forgery with the reason it gets, at the first, second and
last index and on both sides of a slice boundary; memory-mapped files; the model's verdict under fixed challenges; the error
codes; the C++ mode."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from circom_compat_b200 import Groth16, Powers, read_ptau, synth
from circom_compat_b200.zkey import Q_MOD, R_MOD
import ptau_check_model as P
from ptau_model import write_ptau

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLICE = 1 << 22                                    # POWERS_SLICE (csrc/msm.cuh)
NOT_POWERS = "the powers are not those of one tau, alpha and beta"


def _ch(seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R_MOD) for _ in range(5)]


def _copy(c, **fields):
    """a ceremony with the same fields as c (arrays copied), some replaced"""
    arrs = {k: np.array(getattr(c, k), copy=True) for k in P.ARRAYS}
    arrs.update(fields)
    return Powers(c.power, c.power, *(arrs[k] for k in P.ARRAYS))


def _reason(verdict):
    ok, rule, name, index = verdict
    if ok:
        return None
    if rule == 6:
        return NOT_POWERS
    texts = {1: 'a coordinate >= p', 2: 'off the twist' if name in ('tau_g2', 'beta_g2') else 'off the curve', 3: 'at infinity',
             4: 'not in G2', 5: 'not the generator'}
    return f"{name}[{index}]: {texts[rule]}"


def _g2_outside_subgroup():
    from batch_model import twist_point_outside_g2
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % Q_MOD for v in (x0, x1, y0, y1)]).reshape(16)


def _forgeries(c, other):
    """(name, ceremony, reason) for ceremony c of power p and `other`, an honest ceremony of the same power with other secrets;
    each forged entry at index 0, 1 and the last"""
    n = 1 << c.power
    out = []
    for name, last in (('tau_g1', 2 * n - 2), ('tau_g2', n - 1), ('alpha_tau_g1', n - 1), ('beta_tau_g1', n - 1)):
        for i in (0, 1, last):
            a = np.array(getattr(c, name), copy=True)
            a[i] = getattr(other, name)[max(i, 1)]                # a valid point, not the right one
            gen = name in ('tau_g1', 'tau_g2') and i == 0
            out.append((f'{name}[{i}] replaced', _copy(c, **{name: a}), f'{name}[0]: not the generator' if gen else NOT_POWERS))
        for i in (1, last):
            a = np.array(getattr(c, name), copy=True)
            a[i, 4 if name != 'tau_g2' else 8] ^= 1               # the y coordinate's low word
            g2 = name == 'tau_g2'
            out.append((f'{name}[{i}] off its curve', _copy(c, **{name: a}), f"{name}[{i}]: off the {'twist' if g2 else 'curve'}"))
            a = np.array(getattr(c, name), copy=True)
            a[i, 3] = (1 << 64) - 1
            out.append((f'{name}[{i}] coordinate >= p', _copy(c, **{name: a}), f'{name}[{i}]: a coordinate >= p'))
    out.append(('tau_g2 from another tau', _copy(c, tau_g2=np.array(other.tau_g2, copy=True)), NOT_POWERS))
    out.append(('beta_g2 of another beta', _copy(c, beta_g2=np.array(other.beta_g2, copy=True)), NOT_POWERS))
    for i in (1, n - 1):
        a = np.array(c.tau_g2, copy=True)
        a[i] = _g2_outside_subgroup()
        out.append((f'tau_g2[{i}] outside G2', _copy(c, tau_g2=a), f'tau_g2[{i}]: not in G2'))
    out.append(('beta_g2 outside G2', _copy(c, beta_g2=_g2_outside_subgroup().reshape(1, 16)), 'beta_g2[0]: not in G2'))
    a = np.array(c.beta_g2, copy=True); a[0, 9] ^= 1
    out.append(('beta_g2 off its twist', _copy(c, beta_g2=a), 'beta_g2[0]: off the twist'))
    return out


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize('power', [1, 2, 3])
def test_model_accepts_honest_ceremonies(power):
    rng = random.Random(power)
    c = P.CpuCeremony(power, *(rng.randrange(1, R_MOD) for _ in range(3)))
    for k in range(1, power + 1):
        assert P.check(c, k, _ch(k)) == (True, 0, None, None), k


def test_model_accepts_the_new_ceremony():
    """tau = alpha = beta = 1: every point a generator, as `snarkjs powersoftau new` writes it"""
    assert P.check(P.CpuCeremony(2, 1, 1, 1), 2, _ch(3))[0]


def test_model_rejects_each_forgery():
    c, other = P.CpuCeremony(2, 11, 22, 33), P.CpuCeremony(2, 12, 23, 34)
    for name, forged, reason in _forgeries(c, other):
        assert _reason(P.check(forged, 2, _ch(5))) == reason, name
    assert _reason(P.check(P.CpuCeremony(2, 0, 5, 6), 2, _ch(5))) == 'tau_g1[1]: at infinity'
    assert _reason(P.check(P.CpuCeremony(2, 5, 0, 6), 2, _ch(5))) == 'alpha_tau_g1[0]: at infinity'


def test_shifted_sum_identities():
    rng = random.Random(9)
    for m in (2, 3, 7, 16):
        xs = [rng.randrange(R_MOD) for _ in range(m)]
        for rho in (1, 2, R_MOD - 1, rng.randrange(1, R_MOD)):
            direct, from_s = P.shifted_sums(xs, rho)
            assert direct == from_s, (m, rho)


def test_python_entry_refuses_bad_shapes_before_the_library():
    c = P.CpuCeremony(2, 3, 4, 5)
    for log_n in (0, -1, 3):
        with pytest.raises(ValueError):
            Groth16.verify_powers_of_tau(c, log_n=log_n)
    short = Powers(2, 2, c.tau_g1[:6], c.tau_g2, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2)
    with pytest.raises(ValueError, match='tau_g1 holds 6 rows'):
        Groth16.verify_powers_of_tau(short)
    with pytest.raises(ValueError, match='five challenges'):
        Groth16.verify_powers_of_tau(c, challenges=[1, 2, 3])


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope='module')
def gpu():
    from circom_compat_b200 import Context, release_all
    c = Context(0)
    yield c
    release_all()
    c.close()


def _bytes32(vals) -> np.ndarray:
    return np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in vals), dtype='<u8').reshape(-1, 4)


class Ceremony:
    """the arrays of a ceremony of size 2^power for (tau, alpha, beta) on k1 G1 / k2 G2, by fixed-base products"""

    def __init__(self, ctx, power, tau, alpha, beta, k1=1, k2=1):
        n = 1 << power
        self.power = self.ceremony_power = power
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * tau % R_MOD
        self.tau_g1 = ctx.fixed_base_g1(_bytes32([k1 * v % R_MOD for v in t]))
        self.tau_g2 = ctx.fixed_base_g2(_bytes32([k2 * v % R_MOD for v in t[:n]]))
        self.alpha_tau_g1 = ctx.fixed_base_g1(_bytes32([k1 * alpha * v % R_MOD for v in t[:n]]))
        self.beta_tau_g1 = ctx.fixed_base_g1(_bytes32([k1 * beta * v % R_MOD for v in t[:n]]))
        self.beta_g2 = ctx.fixed_base_g2(_bytes32([k2 * beta % R_MOD]))


_CEREMONIES = {}


def _ceremony(ctx, power, seed=7):
    if (power, seed) not in _CEREMONIES:
        rng = random.Random(seed)
        _CEREMONIES[(power, seed)] = Ceremony(ctx, power, *(rng.randrange(1, R_MOD) for _ in range(3)))
    return _CEREMONIES[(power, seed)]


def _powers_scalars(rho, n):
    if rho == 1:
        return np.tile(_bytes32([1]), (n, 1))
    if rho == R_MOD - 1:
        return np.tile(_bytes32([1, R_MOD - 1]), ((n + 1) // 2, 1))[:n]
    out, x = [], 1
    for _ in range(n):
        out.append(x)
        x = x * rho % R_MOD
    return _bytes32(out)


def _bases(ctx, n, g2, seed):
    """n points: 4096 distinct ones tiled (repeated bases), with a few at infinity"""
    rng = random.Random(seed)
    fb = ctx.fixed_base_g2 if g2 else ctx.fixed_base_g1
    base = fb(_bytes32([rng.randrange(1, R_MOD) for _ in range(min(n, 4096))]))
    pts = np.tile(base, ((n + len(base) - 1) // len(base), 1))[:n].copy()
    for i in (n // 2, n - 1, 3):
        if i < n and n > 2:
            pts[i] = 0
    return pts


@pytest.mark.gpu
@pytest.mark.parametrize('g2,n', [(False, 1), (False, 2), (False, 3), (False, 1024), (True, 1), (True, 2), (True, 3), (True, 1024),
                                  (False, SLICE - 1), (False, SLICE), (False, SLICE + 1), (True, SLICE - 1), (True, SLICE),
                                  (True, SLICE + 1), (False, 3 * SLICE + 17)])
def test_powers_msm_matches_the_table_msm(gpu, g2, n):
    pts = _bases(gpu, n, g2, n)
    msm = gpu.msm_g2 if g2 else gpu.msm_g1
    rhos = [random.Random(n).randrange(2, R_MOD)] + ([1, R_MOD - 1] if n <= SLICE + 1 else [])
    for rho in rhos:
        got = gpu.powers_msm(pts, rho, g2=g2)
        assert got.tobytes() == msm(pts, _powers_scalars(rho, n)).tobytes(), (n, rho)
        if n <= 3:
            from oracle import pyref as o
            cur = o.G2 if g2 else o.G1
            want = cur.sum([cur.mul(P.point_of(row, g2)[1], pow(rho, i, R_MOD)) for i, row in enumerate(pts)])
            assert P.point_of(got, g2)[1] == want, (n, rho)
    assert not gpu.powers_msm(pts[:0], 5, g2=g2).any()


@pytest.mark.gpu
@pytest.mark.parametrize('power', [1, 2, 5, 10, 16, 22])
def test_honest_ceremonies_pass(gpu, power):
    c = _ceremony(gpu, power)
    r = Groth16.verify_powers_of_tau(c, ctx=gpu)
    assert r and r.reason is None
    if power == 10:
        for k in range(1, power + 1):
            assert Groth16.verify_powers_of_tau(c, k, gpu), k


@pytest.mark.gpu
def test_the_new_ceremony_passes(gpu):
    assert Groth16.verify_powers_of_tau(Ceremony(gpu, 4, 1, 1, 1), ctx=gpu)


@pytest.mark.gpu
def test_forgeries_are_refused_with_their_reason(gpu):
    c, other = _ceremony(gpu, 5), _ceremony(gpu, 5, seed=8)
    for name, forged, reason in _forgeries(c, other):
        assert Groth16.verify_powers_of_tau(forged, ctx=gpu).reason == reason, name
    assert Groth16.verify_powers_of_tau(Ceremony(gpu, 3, 0, 5, 6), ctx=gpu).reason == 'tau_g1[1]: at infinity'
    assert Groth16.verify_powers_of_tau(Ceremony(gpu, 3, 5, 0, 6), ctx=gpu).reason == 'alpha_tau_g1[0]: at infinity'
    assert Groth16.verify_powers_of_tau(Ceremony(gpu, 3, 5, 6, 7, k1=7), ctx=gpu).reason == 'tau_g1[0]: not the generator'
    assert Groth16.verify_powers_of_tau(Ceremony(gpu, 3, 5, 6, 7, k2=5), ctx=gpu).reason == 'tau_g2[0]: not the generator'


@pytest.mark.gpu
def test_forgeries_on_both_sides_of_a_slice_boundary(gpu):
    """tau_g1 of a power-22 ceremony holds 2^23 - 1 points: the last point of its first slice and the first of its second"""
    c = _ceremony(gpu, 22)
    t = c.tau_g1
    for i in (SLICE - 1, SLICE, 2 * SLICE - 2):
        keep = t[i].copy()
        try:
            t[i] = t[5]
            assert Groth16.verify_powers_of_tau(c, ctx=gpu).reason == NOT_POWERS, i
            t[i] = keep
            t[i, 4] ^= 1
            assert Groth16.verify_powers_of_tau(c, ctx=gpu).reason == f'tau_g1[{i}]: off the curve', i
        finally:
            t[i] = keep
    assert Groth16.verify_powers_of_tau(c, ctx=gpu)


@pytest.mark.gpu
def test_a_prefix_passes_when_the_rest_is_forged(gpu):
    """correct on the points a domain of 2^k reads, forged after them: passes at log_n = k, fails on the whole file"""
    c = _ceremony(gpu, 6)
    for k in (1, 3, 5):
        n = 1 << k
        t = np.array(c.tau_g1, copy=True); t[2 * n - 1] = t[0]
        u = np.array(c.tau_g2, copy=True); u[n] = u[0]
        a = np.array(c.alpha_tau_g1, copy=True); a[n:] = a[0]
        forged = _copy(c, tau_g1=t, tau_g2=u, alpha_tau_g1=a)
        assert Groth16.verify_powers_of_tau(forged, k, gpu), k
        assert Groth16.verify_powers_of_tau(forged, 6, gpu).reason == NOT_POWERS, k


@pytest.mark.gpu
def test_a_memory_mapped_file_gives_the_same_verdict(gpu, tmp_path):
    c = _ceremony(gpu, 10)
    path = tmp_path / 'pot10.ptau'
    path.write_bytes(write_ptau(10, c.tau_g1, c.tau_g2, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2))
    pw = read_ptau(str(path))
    assert isinstance(pw.tau_g1.base, np.ndarray) or pw.tau_g1.base is not None
    for k in (1, 7, 10):
        assert Groth16.verify_powers_of_tau(pw, k, gpu), k
    bad = np.array(c.beta_tau_g1, copy=True); bad[300] = c.beta_tau_g1[301]
    path.write_bytes(write_ptau(10, c.tau_g1, c.tau_g2, c.alpha_tau_g1, bad, c.beta_g2))
    pw = read_ptau(str(path))
    assert Groth16.verify_powers_of_tau(pw, ctx=gpu).reason == NOT_POWERS
    assert Groth16.verify_powers_of_tau(pw, 8, gpu)


@pytest.mark.gpu
def test_fixed_challenges_give_the_models_verdict(gpu):
    c, other = _ceremony(gpu, 2), _ceremony(gpu, 2, seed=8)
    cases = [('honest', _copy(c), None)] + [f for f in _forgeries(c, other) if f[0] in
                                            ('tau_g1[1] replaced', 'tau_g2 from another tau', 'tau_g2[3] outside G2', 'beta_g2 of another beta')]
    for seed in (1, 2):
        ch = _ch(seed)
        for name, cer, _ in cases:
            want = _reason(P.check(cer, 2, ch))
            assert Groth16.verify_powers_of_tau(cer, ctx=gpu, challenges=ch).reason == want, (name, seed)
    # challenges of 1: the equations still hold for an honest ceremony
    assert Groth16.verify_powers_of_tau(c, ctx=gpu, challenges=[1] * 5)


def _raw_check(ctx, cer, log_n, ch=None, log_size=None, null=None):
    from circom_compat_b200 import _native as N
    arrays = {k: np.ascontiguousarray(getattr(cer, k)) for k in P.ARRAYS}
    pd = N.PowersDesc()
    pd.log_size = cer.power if log_size is None else log_size
    for k, a in arrays.items():
        setattr(pd, k, None if k == null else a.ctypes.data)
    cb = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in (ch or _ch(1))), dtype=np.uint8).copy()
    rep = N.PowersReport()
    rc = N.lib().b2g_powers_check(ctx._h, C.byref(pd), log_n, cb.ctypes.data, C.byref(rep))
    return rc, rep


@pytest.mark.gpu
def test_errors_leave_the_context_usable(gpu):
    from circom_compat_b200 import _native as N
    c = _ceremony(gpu, 5)

    def still_usable():
        rc, rep = _raw_check(gpu, c, 5)
        assert rc == N.B2G_OK and rep.ok == 1 and rep.rule == 0

    still_usable()
    cases = [('log_n 0', dict(log_n=0), N.B2G_E_DOMAIN), ('log_n above log_size', dict(log_n=6), N.B2G_E_DOMAIN),
             ('log_size 29', dict(log_n=5, log_size=29), N.B2G_E_DOMAIN),
             ('rho 0', dict(log_n=5, ch=[0, 1, 2, 3, 4]), N.B2G_E_INPUT),
             ('eps r', dict(log_n=5, ch=[1, 2, 3, 4, R_MOD]), N.B2G_E_INPUT),
             ('kappa 2^256 - 1', dict(log_n=5, ch=[1, 2, 3, (1 << 256) - 1, 4]), N.B2G_E_INPUT),
             ('null tau_g2', dict(log_n=5, null='tau_g2'), N.B2G_E_SHAPE)]
    for name, kw, code in cases:
        rc, _ = _raw_check(gpu, c, **kw)
        assert rc == code, (name, rc, N.lib().b2g_last_error())
        still_usable()
    rep = N.PowersReport()
    assert N.lib().b2g_powers_check(gpu._h, None, 5, None, C.byref(rep)) == N.B2G_E_SHAPE
    assert N.lib().b2g_powers_check(None, None, 5, None, None) == N.B2G_E_SHAPE
    out = np.zeros(8, dtype=np.uint64)
    rho = np.frombuffer(R_MOD.to_bytes(32, 'little'), dtype=np.uint8).copy()
    assert N.lib().b2g_powers_msm(gpu._h, 0, 4, c.tau_g1.ctypes.data, rho.ctypes.data, out.ctypes.data) == N.B2G_E_INPUT
    assert N.lib().b2g_powers_msm(gpu._h, 0, 4, None, rho.ctypes.data, out.ctypes.data) == N.B2G_E_SHAPE
    with pytest.raises(N.B2gError):
        Groth16.verify_powers_of_tau(c, ctx=gpu, challenges=[1, 2, 3, 4, 0])
    still_usable()


@pytest.mark.gpu
def test_a_pending_proof_is_refused(gpu):
    from circom_compat_b200 import fr_to_mont, _native as N
    c = _ceremony(gpu, 7)
    circ = synth.chain_circuit(64)
    pk = Groth16.generate_parameters_from_powers_of_tau(circ, c, gpu)
    w = synth.chain_witness(64)
    pending = Groth16.submit(pk, 5, 7, circ.matrices(), fr_to_mont(w), gpu)
    with pytest.raises(N.B2gError, match='pending'):
        Groth16.verify_powers_of_tau(c, ctx=gpu)
    with pytest.raises(N.B2gError, match='pending'):
        gpu.powers_msm(c.tau_g1, 3)
    assert Groth16.verify(pk, w[1:circ.num_inputs], pending.wait())
    assert Groth16.verify_powers_of_tau(c, ctx=gpu)


@pytest.mark.gpu
def test_cpp_ptau_check_mode_matches_python(gpu, tmp_path):
    """B2G_PTAU_CHECK=<file.ptau> groth16_bench [log_n]: the verdict or the reason, as Python gives it"""
    import subprocess
    c = _ceremony(gpu, 8, seed=21)
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    bad = np.array(c.tau_g2, copy=True); bad[17] = _g2_outside_subgroup()
    forged = np.array(c.alpha_tau_g1, copy=True); forged[100] = c.alpha_tau_g1[99]
    files = {'honest': (c.tau_g2, c.alpha_tau_g1), 'not in G2': (bad, c.alpha_tau_g1), 'ratio': (c.tau_g2, forged)}
    for name, (u, a) in files.items():
        path = tmp_path / f'{name}.ptau'
        path.write_bytes(write_ptau(8, c.tau_g1, u, a, c.beta_tau_g1, c.beta_g2))
        for log_n in (None, 6):
            args = [exe] + ([str(log_n)] if log_n else [])
            out = subprocess.check_output(args, text=True, env=dict(os.environ, B2G_PTAU_CHECK=str(path)))
            kv = dict(line.split('=', 1) for line in out.splitlines() if '=' in line)
            want = Groth16.verify_powers_of_tau(read_ptau(str(path)), log_n, gpu)
            assert kv['powers'] == ('1' if want else '0'), (name, log_n, out)
            assert kv.get('reason') == want.reason, (name, log_n, out)
            assert float(kv['ms']) > 0
