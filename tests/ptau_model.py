"""Big-int model of the powers-of-tau setup: a writer of the snarkjs .ptau container (circom_compat_b200/ptau.py restates
the layout), a radix-2 inverse transform over Fr, and the folded CircomReduction H query of b2g_setup_from_powers."""
import struct

import numpy as np

from circom_compat_b200 import synth
from circom_compat_b200.zkey import Q_MOD, R_MOD


def section(sid: int, body: bytes) -> bytes:
    return struct.pack('<IQ', sid, len(body)) + body


def container(sections, magic=b'ptau', version=1) -> bytes:
    """the file of the given (already framed) sections"""
    return magic + struct.pack('<II', version, len(sections)) + b''.join(sections)


def header(power: int, ceremony_power=None, q=Q_MOD, n8=32) -> bytes:
    return section(1, struct.pack('<I', n8) + q.to_bytes(n8, 'little') + struct.pack('<II', power, ceremony_power or power))


def write_ptau(power, tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1, beta_g2, ceremony_power=None) -> bytes:
    """a .ptau file of size 2^power from point arrays (uint64 rows, affine Montgomery), sections 1-6 in order"""
    bodies = [np.ascontiguousarray(a, dtype=np.uint64).tobytes() for a in (tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1, beta_g2)]
    return container([header(power, ceremony_power)] + [section(2 + k, b) for k, b in enumerate(bodies)])


def intt(vals):
    """natural-order inverse radix-2 transform over Fr, scaled by n^-1"""
    n = len(vals)
    w_inv = pow(synth.root_of_unity(n), -1, R_MOD)
    out = _fft([v % R_MOD for v in vals], w_inv)
    ninv = pow(n, -1, R_MOD)
    return [v * ninv % R_MOD for v in out]


def _fft(a, w):
    n = len(a)
    if n == 1:
        return a
    even, odd = _fft(a[0::2], w * w % R_MOD), _fft(a[1::2], w * w % R_MOD)
    out, t = [0] * n, 1
    for k in range(n // 2):
        x = t * odd[k] % R_MOD
        out[k], out[k + n // 2] = (even[k] + x) % R_MOD, (even[k] - x) % R_MOD
        t = t * w % R_MOD
    return out


def folded_circom_h(n: int, tau: int):
    """the discrete logs of the CircomReduction H query as b2g_setup_from_powers computes it: 1/2 iNTT_n(y), with
    y_i = omega_2n^-i (t_i - t_(i+n)), t_i = tau^i for i < 2n - 1 and t_(2n-1) = 0 (infinity)"""
    t = [pow(tau, i, R_MOD) for i in range(2 * n - 1)] + [0]
    w2inv = pow(synth.root_of_unity(2 * n), -1, R_MOD)
    y = [pow(w2inv, i, R_MOD) * (t[i] - t[i + n]) % R_MOD for i in range(n)]
    half = pow(2, -1, R_MOD)
    return [v * half % R_MOD for v in intt(y)]
