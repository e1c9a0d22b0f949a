"""Phase-1 contributions (b2g_powers_contribute, Groth16.contribute_powers_of_tau), the new ceremony (ptau.new_powers_of_tau)
and the per-point product they run (b2g_points_scale).
CPU: the scalar splits of tests/ptau_contribute_model.py and their bounds, the signed-window recoding, the endomorphisms on
points with oracle.pyref, the device constants against the model, the new ceremony, and the Python entry's refusals.
GPU: points_scale against fixed_base byte for byte (and against pyref for n <= 3) across the slice boundary, the device split
against the model, contributions against the ceremony of the products of the secrets (at 22, tau_g1 spans two slices), chains
of contributions, memory-mapped output, the refused inputs and the C++ mode."""
import ctypes as C
import os
import random
import re
import subprocess

import numpy as np
import pytest

from circom_compat_b200 import Groth16, Powers, new_powers_of_tau, read_ptau, write_ptau
from circom_compat_b200.zkey import Q_MOD, R_MOD
import ptau_check_model as P
import ptau_contribute_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLICE = 1 << 22                                    # POWERS_SLICE (csrc/msm.cuh)


def _rand_scalars(seed, count):
    rng = random.Random(seed)
    return [rng.randrange(R_MOD) for _ in range(count)]


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_glv_split_reconstructs_and_is_short():
    for k in M.edge_scalars() + _rand_scalars(1, 10_000):
        k1, k2 = M.glv_split(k)
        assert (k1 + k2 * M.LAMBDA - k) % R_MOD == 0, k
        assert abs(k1) < M.HALF_BOUND and abs(k2) < M.HALF_BOUND, k


def test_gls_split_reconstructs_and_is_short():
    for k in M.edge_scalars() + _rand_scalars(2, 10_000):
        k1, k2 = M.gls_split(k)
        assert k1 + k2 * M.GLS_D == k and 0 <= k1 < M.GLS_D, k
        assert k2 < 1 << 127, k


def test_split_constants():
    assert M.GLS_D == Q_MOD - R_MOD                                 # p = r + 6x^2
    assert (M.LAMBDA ** 2 + M.LAMBDA + 1) % R_MOD == 0 and (M.BETA ** 2 + M.BETA + 1) % Q_MOD == 0
    assert (M.A1 + M.B1 * M.LAMBDA) % R_MOD == 0 and (M.A2 + M.B2 * M.LAMBDA) % R_MOD == 0
    assert M.A1 == M.B2 and M.B1 < 0 < M.B2                       # the device stores A1 once and -B1
    assert max(abs(v) for v in (M.A1, M.B1, M.A2, M.B2)) < 1 << 128


def test_device_constants_match_the_model():
    src = open(os.path.join(ROOT, 'circom_compat_b200', 'csrc', 'contribute.cu')).read()

    def words(name):
        body = re.search(r'__constant__ uint32_t ' + name + r'\[\d+\] = \{([^}]*)\}', src).group(1)
        return sum(int(w.strip().rstrip('u'), 16) << (32 * i) for i, w in enumerate(body.split(',')))
    assert words('SPLIT_BETA') == (M.BETA << 256) % Q_MOD
    assert words('SPLIT_A1') == M.A1 and words('SPLIT_B1') == -M.B1 and words('SPLIT_A2') == M.A2
    assert words('SPLIT_G1R') == M.G1R and words('SPLIT_G2R') == M.G2R
    assert words('SPLIT_D') == M.GLS_D and words('SPLIT_MU') == M.GLS_MU


def test_signed_window_recoding():
    rng = random.Random(3)
    halves = [0, 1, 7, 8, 9, 15, 16, (1 << 127) - 1, 1 << 127, (1 << 128) - 1] + [rng.getrandbits(128) for _ in range(2000)]
    for h in halves:
        d = M.digits(h)
        assert len(d) == M.DIGITS and all(-8 <= x <= 8 for x in d)
        assert sum(x * 16 ** i for i, x in enumerate(d)) == h, h


def test_endomorphisms_on_points():
    from oracle import pairing_model as PM
    from oracle import pyref as o
    assert (M.BETA * o.G1_GEN[0] % Q_MOD, o.G1_GEN[1]) == o.G1.mul(o.G1_GEN, M.LAMBDA)
    assert (M.BETA * o.G1_GEN[0] % Q_MOD, o.G1_GEN[1]) != o.G1.mul(o.G1_GEN, M.LAMBDA * M.LAMBDA % R_MOD)
    for s in (3, 12345, R_MOD - 5):
        p1 = o.G1.mul(o.G1_GEN, s)
        assert (M.BETA * p1[0] % Q_MOD, p1[1]) == o.G1.mul(p1, M.LAMBDA)
        q = o.G2.mul(o.G2_GEN, s)
        assert PM.twist_frobenius(q) == o.G2.mul(q, M.GLS_D)


def test_new_ceremony():
    from circom_compat_b200.groth16 import _mont_points
    from oracle import pyref as o
    c = new_powers_of_tau(3, ceremony_power=9)
    assert (c.power, c.ceremony_power, c.lagrange) == (3, 9, None)
    g1 = _mont_points([o.G1_GEN], False).reshape(8)
    g2 = _mont_points([o.G2_GEN], True).reshape(16)
    assert c.tau_g1.shape == (15, 8) and c.tau_g2.shape == (8, 16) and c.beta_g2.shape == (1, 16)
    for name in P.ARRAYS:
        a = np.asarray(getattr(c, name))
        assert (a == (g2 if a.shape[1] == 16 else g1)).all(), name
    buf = __import__('io').BytesIO()
    write_ptau(buf, c)
    back = read_ptau(buf.getvalue())
    assert (back.power, back.ceremony_power) == (3, 9)
    for name in P.ARRAYS:
        assert np.array_equal(getattr(back, name), getattr(c, name)), name
    assert P.check(c, 3, [5, 6, 7, 8, 9]) == (True, 0, None, None)
    with pytest.raises(ValueError):
        new_powers_of_tau(0)
    with pytest.raises(ValueError):
        new_powers_of_tau(29)


def test_python_entry_refuses_before_the_library():
    from circom_compat_b200 import B2gError
    c = new_powers_of_tau(2)
    short = Powers(2, 2, c.tau_g1[:6], c.tau_g2, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2)
    with pytest.raises(ValueError, match='tau_g1 holds 6 rows'):
        Groth16.contribute_powers_of_tau(short, tau=2, alpha=3, beta=4)
    for bad in (0, R_MOD, R_MOD + 1):
        for name in ('tau', 'alpha', 'beta'):
            with pytest.raises(B2gError, match=f'secret {name} is 0 or >= r') as e:
                Groth16.contribute_powers_of_tau(c, **{'tau': 2, 'alpha': 3, 'beta': 4, name: bad})
            assert e.value.code == -4
    for power in (0, 29):
        with pytest.raises(ValueError, match='outside 1..28'):
            Groth16.contribute_powers_of_tau(Powers(power, power, c.tau_g1, c.tau_g2, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2))


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
    """the arrays of a ceremony of size 2^power for (tau, alpha, beta), by fixed-base products"""

    def __init__(self, ctx, power, tau, alpha, beta):
        n = 1 << power
        self.power = self.ceremony_power = power
        self.lagrange = None
        t = [1] * (2 * n - 1)
        for i in range(1, 2 * n - 1):
            t[i] = t[i - 1] * tau % R_MOD
        self.tau_g1 = ctx.fixed_base_g1(_bytes32(t))
        self.tau_g2 = ctx.fixed_base_g2(_bytes32(t[:n]))
        self.alpha_tau_g1 = ctx.fixed_base_g1(_bytes32([alpha * v % R_MOD for v in t[:n]]))
        self.beta_tau_g1 = ctx.fixed_base_g1(_bytes32([beta * v % R_MOD for v in t[:n]]))
        self.beta_g2 = ctx.fixed_base_g2(_bytes32([beta % R_MOD]))


def _same(a, b):
    for name in P.ARRAYS:
        x, y = np.asarray(getattr(a, name)), np.asarray(getattr(b, name))
        assert x.shape == y.shape and np.array_equal(x, y), name


def _edge_k():
    return [0, 1, R_MOD - 1, M.LAMBDA, M.GLS_D, 1 << 127, (1 << 128) - 1, (1 << 128) + 1, 2, M.LAMBDA + 1, M.GLS_D - 1]


@pytest.mark.gpu
@pytest.mark.parametrize('g2', [False, True])
@pytest.mark.parametrize('n', [1, 2, 3, 1024, SLICE - 1, SLICE, SLICE + 1])
def test_points_scale_matches_fixed_base(gpu, g2, n):
    """P_i = s_i G, k_i with the edge scalars: points_scale(P, k)_i == fixed_base(s_i k_i); a few P_i at infinity"""
    rng = random.Random(n * 2 + g2)
    period = min(n, 4096)
    s = [rng.randrange(1, R_MOD) for _ in range(period)]
    k = [rng.randrange(R_MOD) for _ in range(period)]
    edge = _edge_k()
    for j in range(period):
        if j % 3 == 0:
            k[j] = edge[(j // 3) % len(edge)]
    inf = {j for j in (1, period // 2) if j < period and period > 2}
    fb = gpu.fixed_base_g2 if g2 else gpu.fixed_base_g1
    base = fb(_bytes32(s))
    want1 = fb(_bytes32([s[j] * k[j] % R_MOD for j in range(period)]))
    for j in inf:
        base[j] = 0
        want1[j] = 0
    reps = (n + period - 1) // period
    pts = np.tile(base, (reps, 1))[:n]
    ks = np.tile(_bytes32(k), (reps, 1))[:n]
    got = gpu.points_scale(pts, ks, g2=g2)
    want = np.tile(want1, (reps, 1))[:n]
    assert np.array_equal(got, want)
    if n <= 3:
        from oracle import pyref as o
        curve = o.G2 if g2 else o.G1
        for i in range(n):
            p = P.point_of(pts[i], g2)[1]
            exp = None if p is None else curve.mul(p, k[i])
            assert P.point_of(got[i], g2)[1] == exp, i


@pytest.mark.gpu
def test_points_scale_refuses_a_scalar_not_below_r(gpu):
    from circom_compat_b200 import B2gError
    pts = gpu.fixed_base_g1(_bytes32([3, 4]))
    with pytest.raises(B2gError, match=r'scalars\[1\] is not below r') as e:
        gpu.points_scale(pts, _bytes32([5, R_MOD]))
    assert e.value.code == -4
    assert np.array_equal(gpu.points_scale(pts, _bytes32([1, 1])), pts)


@pytest.mark.gpu
def test_device_split_matches_the_model(gpu):
    ks = M.edge_scalars() + _rand_scalars(4, 4096)
    out = gpu.test_op(54, _bytes32(ks))
    raw = out.astype('<u8').tobytes()
    for i, k in enumerate(ks):
        vals = []
        for h in range(4):
            v = int.from_bytes(raw[128 * i + 32 * h:128 * i + 32 * h + 32], 'little')
            vals.append(v - (1 << 256) if v >> 255 else v)
        assert tuple(vals[:2]) == M.glv_split(k), k
        assert tuple(vals[2:]) == M.gls_split(k), k


_SECRETS = (0x1234567 * 10 ** 40 % R_MOD, R_MOD - 3, 987654321)


@pytest.mark.gpu
@pytest.mark.parametrize('power', [1, 2, 5, 10, 16, 22])
def test_contribution_is_the_ceremony_of_the_products(gpu, power):
    rng = random.Random(power)
    tau, alpha, beta = (rng.randrange(1, R_MOD) for _ in range(3))
    t, a, b = (rng.randrange(1, R_MOD) for _ in range(3))
    before = Ceremony(gpu, power, tau, alpha, beta)
    after = Groth16.contribute_powers_of_tau(before, ctx=gpu, tau=t, alpha=a, beta=b)
    assert (after.power, after.ceremony_power, after.lagrange) == (power, power, None)
    _same(after, Ceremony(gpu, power, tau * t % R_MOD, alpha * a % R_MOD, beta * b % R_MOD))
    assert Groth16.verify_powers_of_tau(after, ctx=gpu)


@pytest.mark.gpu
@pytest.mark.parametrize('power', [1, 4, 10])
def test_new_contributions_chains_and_identity(gpu, power):
    t, a, b = _SECRETS
    first = Groth16.contribute_powers_of_tau(new_powers_of_tau(power), ctx=gpu, tau=t, alpha=a, beta=b)
    _same(first, Ceremony(gpu, power, t, a, b))
    assert Groth16.verify_powers_of_tau(first, ctx=gpu)
    t2, a2, b2 = 5, R_MOD - 1, 1 << 200
    second = Groth16.contribute_powers_of_tau(first, ctx=gpu, tau=t2, alpha=a2, beta=b2)
    _same(second, Groth16.contribute_powers_of_tau(new_powers_of_tau(power), ctx=gpu, tau=t * t2 % R_MOD, alpha=a * a2 % R_MOD,
                                                   beta=b * b2 % R_MOD))
    assert Groth16.verify_powers_of_tau(second, ctx=gpu)
    _same(Groth16.contribute_powers_of_tau(second, ctx=gpu, tau=1, alpha=1, beta=1), second)
    drawn = Groth16.contribute_powers_of_tau(first, ctx=gpu, rng=random.Random(1))
    assert Groth16.verify_powers_of_tau(drawn, ctx=gpu)


@pytest.mark.gpu
def test_memory_mapped_output(gpu, tmp_path):
    c = Groth16.contribute_powers_of_tau(new_powers_of_tau(6, ceremony_power=12), ctx=gpu, tau=7, alpha=8, beta=9)
    prepared = Groth16.prepare_powers_of_tau(c, ctx=gpu)
    assert prepared.lagrange is not None
    mem = Groth16.contribute_powers_of_tau(prepared, ctx=gpu, tau=11, alpha=12, beta=13)
    dst = tmp_path / 'out.ptau'
    got = Groth16.contribute_powers_of_tau(prepared, dst=dst, ctx=gpu, tau=11, alpha=12, beta=13)
    assert (got.power, got.ceremony_power, got.lagrange) == (6, 12, None)
    assert (mem.ceremony_power, mem.lagrange) == (12, None)
    _same(got, mem)
    _same(read_ptau(str(dst)), mem)
    assert Groth16.verify_powers_of_tau(got, ctx=gpu)


def _g2_outside_subgroup():
    from batch_model import twist_point_outside_g2
    from circom_compat_b200 import synth
    (x0, x1), (y0, y1) = twist_point_outside_g2(random.Random(5))
    return synth._ints_to_limbs([v * (1 << 256) % Q_MOD for v in (x0, x1, y0, y1)]).reshape(16)


def _with(c, **fields):
    arrs = {k: np.array(getattr(c, k), copy=True) for k in P.ARRAYS}
    arrs.update(fields)
    return Powers(c.power, c.power, *(arrs[k] for k in P.ARRAYS))


def _refusals(c):
    n = 1 << c.power
    out = []
    a = np.array(c.alpha_tau_g1, copy=True); a[3, 4] ^= 1
    out.append((_with(c, alpha_tau_g1=a), 'alpha_tau_g1[3]: off the curve'))
    a = np.array(c.tau_g2, copy=True); a[n - 1, 8] ^= 1
    out.append((_with(c, tau_g2=a), f'tau_g2[{n - 1}]: off the twist'))
    a = np.array(c.beta_tau_g1, copy=True); a[2, 3] = (1 << 64) - 1
    out.append((_with(c, beta_tau_g1=a), 'beta_tau_g1[2]: a coordinate >= p'))
    a = np.array(c.tau_g1, copy=True); a[2 * n - 2] = 0
    out.append((_with(c, tau_g1=a), f'tau_g1[{2 * n - 2}]: at infinity'))
    a = np.array(c.tau_g1, copy=True); a[0] = c.tau_g1[1]
    out.append((_with(c, tau_g1=a), 'tau_g1[0]: not the generator'))
    a = np.array(c.tau_g2, copy=True); a[0] = c.tau_g2[1]
    out.append((_with(c, tau_g2=a), 'tau_g2[0]: not the generator'))
    for i in (1, n - 1):
        a = np.array(c.tau_g2, copy=True); a[i] = _g2_outside_subgroup()
        out.append((_with(c, tau_g2=a), f'tau_g2[{i}]: not in G2'))
    out.append((_with(c, beta_g2=_g2_outside_subgroup().reshape(1, 16)), 'beta_g2[0]: not in G2'))
    return out


@pytest.mark.gpu
def test_refused_inputs_leave_the_context_usable(gpu):
    from circom_compat_b200 import B2gError
    c = Ceremony(gpu, 4, 3, 5, 7)
    for bad, reason in _refusals(c):
        with pytest.raises(B2gError, match=re.escape(reason)) as e:
            Groth16.contribute_powers_of_tau(bad, ctx=gpu, tau=2, alpha=3, beta=4)
        assert e.value.code == -4, reason
    _same(Groth16.contribute_powers_of_tau(c, ctx=gpu, tau=2, alpha=3, beta=4), Ceremony(gpu, 4, 6, 15, 28))


@pytest.mark.gpu
def test_g2_outside_the_subgroup_across_a_slice_boundary(gpu):
    from circom_compat_b200 import B2gError
    c = new_powers_of_tau(22)
    u = np.array(c.tau_g2, copy=True)
    u[SLICE - 1] = _g2_outside_subgroup()
    bad = Powers(22, 22, c.tau_g1, u, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2)
    with pytest.raises(B2gError, match=re.escape(f'tau_g2[{SLICE - 1}]: not in G2')):
        Groth16.contribute_powers_of_tau(bad, ctx=gpu, tau=2, alpha=3, beta=4)
    t1 = np.array(c.tau_g1, copy=True)
    t1[SLICE + 5] = 0
    bad = Powers(22, 22, t1, c.tau_g2, c.alpha_tau_g1, c.beta_tau_g1, c.beta_g2)
    with pytest.raises(B2gError, match=re.escape(f'tau_g1[{SLICE + 5}]: at infinity')):
        Groth16.contribute_powers_of_tau(bad, ctx=gpu, tau=2, alpha=3, beta=4)


@pytest.mark.gpu
def test_library_refusals(gpu):
    """the C entry's own refusals: secrets 0 and >= r (B2G_E_INPUT), the domain, null pointers, an aliased output"""
    from circom_compat_b200 import _native as N
    from circom_compat_b200.groth16 import _c
    c = new_powers_of_tau(2)
    keep = [_c(getattr(c, k)) for k in P.ARRAYS]
    pd = N.PowersDesc()
    pd.log_size = 2
    for name, a in zip(P.ARRAYS, keep):
        setattr(pd, name, a.ctypes.data)
    outs = [np.zeros_like(a) for a in keep]
    od = N.PowersOut()
    for name, a in zip(P.ARRAYS, outs):
        setattr(od, name, a.ctypes.data)

    def call(vals, desc=pd, out=od):
        sb = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in vals), dtype=np.uint8).copy()
        sd = N.PowersSecrets()
        sd.tau, sd.alpha, sd.beta = sb.ctypes.data, sb.ctypes.data + 32, sb.ctypes.data + 64
        rc = N.lib().b2g_powers_contribute(gpu._h, C.byref(desc), C.byref(sd), C.byref(out))
        return rc, N.lib().b2g_last_error().decode()
    assert call((0, 1, 1)) == (N.B2G_E_INPUT, 'secret tau is 0 or >= r')
    assert call((1, R_MOD, 1)) == (N.B2G_E_INPUT, 'secret alpha is 0 or >= r')
    assert call((1, 1, (1 << 256) - 1)) == (N.B2G_E_INPUT, 'secret beta is 0 or >= r')
    for p in (0, 29):
        d = N.PowersDesc.from_buffer_copy(pd)
        d.log_size = p
        assert call((2, 3, 4), desc=d)[0] == N.B2G_E_DOMAIN
    o = N.PowersOut.from_buffer_copy(od)
    o.beta_g2 = None
    assert call((2, 3, 4), out=o)[0] == N.B2G_E_SHAPE
    o = N.PowersOut.from_buffer_copy(od)
    o.tau_g2 = keep[1].ctypes.data
    assert call((2, 3, 4), out=o)[0] == N.B2G_E_SHAPE
    assert call((2, 3, 4)) == (N.B2G_OK, call((2, 3, 4))[1])
    _same(Powers(2, 2, *outs), Ceremony(gpu, 2, 2, 3, 4))


@pytest.mark.gpu
def test_pending_proof_is_refused(gpu, test_zkey_bytes, golden):
    from circom_compat_b200 import B2gError, fr_to_mont, read_zkey
    pk, cm = read_zkey(test_zkey_bytes)
    g = golden['test_zkey']
    pending = Groth16.submit(pk, int(g['proofs'][0]['r']), int(g['proofs'][0]['s']), cm, fr_to_mont([int(x) for x in g['witness']]), gpu)
    try:
        with pytest.raises(B2gError, match='pending') as e:
            Groth16.contribute_powers_of_tau(new_powers_of_tau(2), ctx=gpu, tau=2, alpha=3, beta=4)
        assert e.value.code == -2
        with pytest.raises(B2gError, match='pending'):
            gpu.points_scale(gpu.fixed_base_g1(_bytes32([3])), [5])
    finally:
        pending.wait()
    Groth16.contribute_powers_of_tau(new_powers_of_tau(2), ctx=gpu, tau=2, alpha=3, beta=4)


@pytest.mark.gpu
def test_cpp_contribute_mode_matches_python(gpu, tmp_path):
    """B2G_PTAU_CONTRIBUTE=<in.ptau> groth16_bench <out.ptau> tau alpha beta writes the file Python writes"""
    exe = os.path.join(ROOT, 'circom_compat_b200', 'host', 'groth16_bench')
    src = tmp_path / 'in.ptau'
    write_ptau(str(src), Ceremony(gpu, 5, 3, 5, 7))
    t, a, b = _SECRETS
    py = tmp_path / 'py.ptau'
    Groth16.contribute_powers_of_tau(read_ptau(str(src)), dst=py, ctx=gpu, tau=t, alpha=a, beta=b)
    cpp = tmp_path / 'cpp.ptau'
    out = subprocess.check_output([exe, str(cpp), str(t), str(a), str(b)], text=True,
                                  env=dict(os.environ, B2G_PTAU_CONTRIBUTE=str(src)))
    assert 'power=5' in out
    assert cpp.read_bytes() == py.read_bytes()
