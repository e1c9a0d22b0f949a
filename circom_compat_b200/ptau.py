"""Reader of snarkjs powers-of-tau ceremony files (.ptau), the phase-1 input of `snarkjs groth16 setup`.

The container, as the reader checks it (DESIGN.md restates it):
    magic b'ptau', u32 version (1), u32 number of sections; then per section a u32 id, a u64 size and its content.
    section 1: u32 n8 (32), q (n8 bytes, BN254's base field), u32 power p, u32 ceremony power
    section 2: tau_g1       = tau^i G1,        i < 2^(p+1) - 1
    section 3: tau_g2       = tau^i G2,        i < 2^p
    section 4: alpha_tau_g1 = alpha tau^i G1,  i < 2^p
    section 5: beta_tau_g1  = beta tau^i G1,   i < 2^p
    section 6: beta_g2      = beta G2 (one point)
Points are Montgomery little-endian, G1 = x, y (64 B) and G2 = x.c0, x.c1, y.c0, y.c1 (128 B), as in a .zkey; all-zero is
infinity.  The prepared Lagrange sections 12-15 are not read: b2g_setup_from_powers transforms the monomial powers itself.

read_ptau returns zero-copy views of sections 2-6 over the file's memory map (or over the given bytes), as rows of 8 / 16
uint64 words, the b2g_pk_desc layout.  Nothing is read beyond the headers until a caller touches the points, and the setup
reads only the prefix its circuit needs, so a ceremony file much larger than memory serves small circuits.

PowersCheck is the verdict of Groth16.verify_powers_of_tau (b2g_powers_check): truthy when the ceremony passes, with the
reason of a failure in the messages b2g_setup_from_powers uses ("tau_g2[17]: not in G2").
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np

from .zkey import Q_MOD

_G1, _G2 = 64, 128
_MAX_POWER = 28


@dataclass
class Powers:
    """the points of a ceremony of size 2^power (views; rows of 8 / 16 uint64 words, affine Montgomery)"""
    power: int
    ceremony_power: int
    tau_g1: np.ndarray
    tau_g2: np.ndarray
    alpha_tau_g1: np.ndarray
    beta_tau_g1: np.ndarray
    beta_g2: np.ndarray

    def prefix(self, log_n: int, copy: bool = False) -> 'Powers':
        """the points a circuit of domain 2^log_n reads (2n - 1 / n / n / n / 1), as views or, with copy, in host memory;
        raises ValueError when the arrays hold fewer points or log_n exceeds the power"""
        if not 0 <= log_n <= self.power:
            raise ValueError(f"ptau: a domain of 2^{log_n} points exceeds the ceremony's 2^{self.power}")
        n = 1 << log_n
        out = []
        for name, count, words in (('tau_g1', 2 * n - 1, 8), ('tau_g2', n, 16), ('alpha_tau_g1', n, 8), ('beta_tau_g1', n, 8),
                                   ('beta_g2', 1, 16)):
            a = np.asarray(getattr(self, name))
            if a.ndim != 2 or a.shape[1] != words or a.shape[0] < count:
                raise ValueError(f"ptau: {name} holds {a.shape[0] if a.ndim == 2 else a.size} rows of "
                                 f"{a.shape[-1] if a.ndim else 0} words; a domain of {n} points reads {count} rows of {words}")
            a = a[:count]
            out.append(np.array(a, dtype=np.uint64, order='C', copy=True) if copy else a)
        return Powers(self.power, self.ceremony_power, *out)


ARRAYS = ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')
NOT_POWERS = "the powers are not those of one tau, alpha and beta"
# b2g_powers_report rule codes 1-5 (G1 text, G2 text)
_RULES = {1: ('a coordinate >= p',) * 2, 2: ('off the curve', 'off the twist'), 3: ('at infinity',) * 2, 4: ('not in G2',) * 2,
          5: ('not the generator',) * 2}


@dataclass
class PowersCheck:
    """the verdict of a ceremony check: truthy when it passes.  rule (b2g_powers_report): 0 ok, 1 a coordinate >= p, 2 off its
    curve, 3 at infinity, 4 outside G2, 5 not the generator (array / index name the point), 6 the ratio rules fail"""
    ok: bool
    rule: int = 0
    array: str = None
    index: int = None

    def __bool__(self) -> bool:
        return bool(self.ok)

    @property
    def reason(self):
        if self.ok:
            return None
        if self.rule == 6:
            return NOT_POWERS
        return f"{self.array}[{self.index}]: {_RULES[self.rule][self.array in ('tau_g2', 'beta_g2')]}"


def _buffer(src) -> np.ndarray:
    if isinstance(src, (str, os.PathLike)):
        if os.path.getsize(src) == 0:
            raise ValueError("ptau: the file is empty")
        return np.memmap(src, dtype=np.uint8, mode='r')
    if isinstance(src, (bytes, bytearray, memoryview)):
        return np.frombuffer(src, dtype=np.uint8)
    if isinstance(src, np.ndarray):
        return src.view(np.uint8).reshape(-1)
    raise TypeError("read_ptau takes a path, bytes or a uint8 array")


def _u32(buf, at) -> int:
    return int.from_bytes(buf[at:at + 4].tobytes(), 'little')


def read_ptau(src) -> Powers:
    """Parse a snarkjs .ptau container: `src` is a path (memory-mapped), bytes or a uint8 array.  Raises ValueError, naming the
    problem, for a wrong magic or version, a field other than BN254's, a missing or truncated section, or a section whose size
    disagrees with the power."""
    buf = _buffer(src)
    size = buf.size
    if size < 12 or buf[:4].tobytes() != b'ptau':
        raise ValueError("ptau: bad magic (not a .ptau file)")
    version = _u32(buf, 4)
    if version != 1:
        raise ValueError(f"ptau: unsupported version {version} (expected 1)")
    n_sections = _u32(buf, 8)
    sections, at = {}, 12
    for k in range(n_sections):
        if at + 12 > size:
            raise ValueError(f"ptau: section header {k} is truncated")
        sid = _u32(buf, at)
        length = int.from_bytes(buf[at + 4:at + 12].tobytes(), 'little')
        at += 12
        if at + length > size:
            raise ValueError(f"ptau: section {sid} is truncated ({length} bytes declared, {size - at} left)")
        sections.setdefault(sid, (at, length))
        at += length
    for sid in range(1, 7):
        if sid not in sections:
            raise ValueError(f"ptau: section {sid} is missing")
    at, length = sections[1]
    if length < 4:
        raise ValueError("ptau: section 1 is truncated")
    n8 = _u32(buf, at)
    if n8 != 32:
        raise ValueError(f"ptau: field element size {n8} is not BN254's (32)")
    if length != 4 + n8 + 8:
        raise ValueError(f"ptau: section 1 holds {length} bytes, not {4 + n8 + 8}")
    q = int.from_bytes(buf[at + 4:at + 36].tobytes(), 'little')
    if q != Q_MOD:
        raise ValueError("ptau: the curve's base field is not BN254's")
    power, ceremony_power = _u32(buf, at + 36), _u32(buf, at + 40)
    if not 1 <= power <= _MAX_POWER:
        raise ValueError(f"ptau: power {power} is out of range (1..{_MAX_POWER})")
    counts = {2: (2 << power) - 1, 3: 1 << power, 4: 1 << power, 5: 1 << power, 6: 1}
    rows = {2: _G1, 3: _G2, 4: _G1, 5: _G1, 6: _G2}
    views = {}
    for sid, count in counts.items():
        at, length = sections[sid]
        if length != count * rows[sid]:
            raise ValueError(f"ptau: section {sid} holds {length} bytes, but power {power} needs {count * rows[sid]}")
        views[sid] = buf[at:at + length].view('<u8').reshape(count, rows[sid] // 8)
    return Powers(power, ceremony_power, views[2], views[3], views[4], views[5], views[6])
