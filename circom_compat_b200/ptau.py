"""Reader of snarkjs powers-of-tau ceremony files (.ptau), the phase-1 input of `snarkjs groth16 setup`.

The container, as the reader checks it (DESIGN.md restates it):
    magic b'ptau', u32 version (1), u32 number of sections; then per section a u32 id, a u64 size and its content.
    section 1: u32 n8 (32), q (n8 bytes, BN254's base field), u32 power p, u32 ceremony power
    section 2: tau_g1       = tau^i G1,        i < 2^(p+1) - 1
    section 3: tau_g2       = tau^i G2,        i < 2^p
    section 4: alpha_tau_g1 = alpha tau^i G1,  i < 2^p
    section 5: beta_tau_g1  = beta tau^i G1,   i < 2^p
    section 6: beta_g2      = beta G2 (one point)
    section 12: lagrange_tau_g1, blocks k = 0 .. p + 1 (2^(p+2) - 1 points)    section 13: lagrange_tau_g2, blocks k = 0 .. p
    section 14: lagrange_alpha_tau_g1, blocks k = 0 .. p                         section 15: lagrange_beta_tau_g1, k = 0 .. p
Points are Montgomery little-endian, G1 = x, y (64 B) and G2 = x.c0, x.c1, y.c0, y.c1 (128 B), as in a .zkey; all-zero is
infinity.  Sections 12-15 are what `snarkjs powersoftau prepare phase2` adds: block k starts at point 2^k - 1 and holds
iNTT_(2^k) of the first 2^k points of the matching monomial section (natural order, scaled by 2^-k), so entry i is L_i(tau)
times the base point for the domain of 2^k points.  The top block of section 12 has only 2^(p+1) - 1 powers to work from and
transforms (tau_g1[0 .. 2^(p+1) - 1), infinity).  The reader attaches them as Powers.lagrange only when all four are present
with the sizes the power implies; otherwise lagrange is None and the Lagrange sections are ignored.

read_ptau returns zero-copy views of sections 2-6 (and 12-15) over the file's memory map (or over the given bytes), as rows of 8 / 16
uint64 words, the b2g_pk_desc layout.  Nothing is read beyond the headers until a caller touches the points, and the setup
reads only the prefix its circuit needs, so a ceremony file much larger than memory serves small circuits.  write_ptau
streams a Powers back into a container, sections 12-15 included when it carries them.

PowersCheck is the verdict of Groth16.verify_powers_of_tau (b2g_powers_check): truthy when the ceremony passes, with the
reason of a failure in the messages b2g_setup_from_powers uses ("tau_g2[17]: not in G2").
"""
from __future__ import annotations

import os
import struct
from dataclasses import dataclass

import numpy as np

from .zkey import Q_MOD

_G1, _G2 = 64, 128
_MAX_POWER = 28
LAGRANGE = ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1')
_LAGRANGE_IDS = (12, 13, 14, 15)


def lagrange_counts(power: int) -> tuple:
    """the points of sections 12-15 of a prepared ceremony of power p: blocks 0 .. p + 1 of G1, then blocks 0 .. p"""
    return ((4 << power) - 1, (2 << power) - 1, (2 << power) - 1, (2 << power) - 1)


@dataclass
class Lagrange:
    """sections 12-15 of a ceremony prepared at `power` (views; rows of 8 / 16 uint64 words, affine Montgomery): block k of a
    section starts at row 2^k - 1 and holds iNTT_(2^k) of the first 2^k points of the monomial section of the same name.
    Block power + 1 of tau_g1 transforms (tau_g1[0 .. 2^(power+1) - 1), infinity); a prefix keeps `power` and fewer blocks."""
    power: int
    tau_g1: np.ndarray
    tau_g2: np.ndarray
    alpha_tau_g1: np.ndarray
    beta_tau_g1: np.ndarray


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
    lagrange: Lagrange = None

    def prefix(self, log_n: int, copy: bool = False) -> 'Powers':
        """the points a circuit of domain 2^log_n reads (2n - 1 / n / n / n / 1), as views or, with copy, in host memory;
        raises ValueError when the arrays hold fewer points or log_n exceeds the power.  The Lagrange sections, when present,
        keep blocks up to log_n + 1 in tau_g1 and up to log_n in the others.  Below the prepared power their top tau_g1 block
        transforms 2n powers, so the prefix then keeps 2n rows of tau_g1 (the last one is what that block reads)."""
        if not 0 <= log_n <= self.power:
            raise ValueError(f"ptau: a domain of 2^{log_n} points exceeds the ceremony's 2^{self.power}")
        n = 1 << log_n
        lag = self.lagrange
        t1 = 2 * n if lag is not None and log_n < lag.power else 2 * n - 1
        out = [_rows_of(getattr(self, name), name, count, words, n, copy)
               for name, count, words in (('tau_g1', t1, 8), ('tau_g2', n, 16), ('alpha_tau_g1', n, 8), ('beta_tau_g1', n, 8),
                                          ('beta_g2', 1, 16))]
        if lag is not None:
            if log_n > lag.power:
                raise ValueError(f"ptau: a domain of 2^{log_n} points exceeds the Lagrange sections' 2^{lag.power}")
            counts = lagrange_counts(log_n)
            lag = Lagrange(lag.power, *(_rows_of(getattr(lag, name), 'lagrange_' + name, c, 16 if name == 'tau_g2' else 8, n, copy)
                                        for name, c in zip(LAGRANGE, counts)))
        return Powers(self.power, self.ceremony_power, *out, lagrange=lag)


def _rows_of(a, name, count, words, n, copy):
    a = np.asarray(a)
    if a.ndim != 2 or a.shape[1] != words or a.shape[0] < count:
        raise ValueError(f"ptau: {name} holds {a.shape[0] if a.ndim == 2 else a.size} rows of "
                         f"{a.shape[-1] if a.ndim else 0} words; a domain of {n} points reads {count} rows of {words}")
    a = a[:count]
    return np.array(a, dtype=np.uint64, order='C', copy=True) if copy else a


ARRAYS = ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')
# b2g_powers_report array codes: ARRAYS, then the Lagrange sections 12-15
REPORT_ARRAYS = ARRAYS + tuple('lagrange_' + k for k in LAGRANGE)
NOT_POWERS = "the powers are not those of one tau, alpha and beta"
# b2g_powers_report rule codes 1-5 (G1 text, G2 text)
_RULES = {1: ('a coordinate >= p',) * 2, 2: ('off the curve', 'off the twist'), 3: ('at infinity',) * 2, 4: ('not in G2',) * 2,
          5: ('not the generator',) * 2}


@dataclass
class PowersCheck:
    """the verdict of a ceremony check: truthy when it passes.  rule (b2g_powers_report): 0 ok, 1 a coordinate >= p, 2 off its
    curve, 3 at infinity, 4 outside G2, 5 not the generator (array / index name the point), 6 the ratio rules fail, 7 the
    Lagrange section `array` is not the transform of its monomial section"""
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
        if self.rule == 7:
            return f"{self.array} is not the transform of {self.array[len('lagrange_'):]}"
        return f"{self.array}[{self.index}]: {_RULES[self.rule][self.array in ('tau_g2', 'beta_g2', 'lagrange_tau_g2')]}"


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
    lagrange = None
    lag_rows = dict(zip(_LAGRANGE_IDS, (_G1, _G2, _G1, _G1)))
    lag_counts = dict(zip(_LAGRANGE_IDS, lagrange_counts(power)))
    if all(sid in sections and sections[sid][1] == lag_counts[sid] * lag_rows[sid] for sid in _LAGRANGE_IDS):
        lagrange = Lagrange(power, *(buf[sections[sid][0]:sections[sid][0] + sections[sid][1]].view('<u8')
                                     .reshape(lag_counts[sid], lag_rows[sid] // 8) for sid in _LAGRANGE_IDS))
    return Powers(power, ceremony_power, views[2], views[3], views[4], views[5], views[6], lagrange)


def _generator_rows():
    """the standard generators G1 = (1, 2) and G2 as one Montgomery row of 8 / 16 words each"""
    from .zkey import Q_MOD
    g2 = ((0x1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed,
           0x198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2),
          (0x12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa,
           0x090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b))
    enc = lambda vals: np.frombuffer(b''.join(((v << 256) % Q_MOD).to_bytes(32, 'little') for v in vals), dtype='<u8').copy()
    return enc((1, 2)), enc((g2[0][0], g2[0][1], g2[1][0], g2[1][1]))


def new_powers_of_tau(power: int, ceremony_power: int = None) -> Powers:
    """`snarkjs powersoftau new`: the ceremony of power p before any contribution, tau = alpha = beta = 1, so every point is
    the generator.  The arrays are read-only zero-copy broadcasts of one row (write_ptau streams them to a file;
    Groth16.contribute_powers_of_tau reads them).  ceremony_power (default p) is kept in section 1."""
    p = int(power)
    if not 1 <= p <= _MAX_POWER:
        raise ValueError(f"ptau: power {p} is out of range (1..{_MAX_POWER})")
    cp = p if ceremony_power is None else int(ceremony_power)
    g1, g2 = _generator_rows()
    n = 1 << p
    return Powers(p, cp, np.broadcast_to(g1, (2 * n - 1, 8)), np.broadcast_to(g2, (n, 16)), np.broadcast_to(g1, (n, 8)),
                  np.broadcast_to(g1, (n, 8)), np.broadcast_to(g2, (1, 16)))


_WRITE_CHUNK = 1 << 26                                  # bytes per write: a file far larger than memory streams through


def write_ptau(dst, powers: Powers, lagrange_space: bool = False, points_space: bool = False) -> None:
    """Write `powers` as a snarkjs .ptau container at the path `dst` (or into a writable binary file object): sections 1-6,
    then 12-15 when powers.lagrange is set.  The arrays must hold the full counts of powers.power (2^(p+1) - 1 / 2^p / 2^p /
    2^p / 1 points, and lagrange_counts(p) with lagrange.power = p); a prefix of a larger ceremony is refused with a
    ValueError.  The points are copied in pieces of 64 MiB, so memory-mapped arrays of any size stream to disk.  Section 7,
    the contribution transcript, is not written: this library neither produces nor checks it, and a reader that needs it (a
    `snarkjs powersoftau verify`) refuses the file.  With lagrange_space and no powers.lagrange, sections 12-15 are written as
    zero-filled space (sparse where the file system allows) for a caller that fills them in place through a memory map, as
    Groth16.prepare_powers_of_tau does.  With points_space, sections 2-6 are written the same way, as space for the
    counts of powers.power (their arrays are not read), for Groth16.contribute_powers_of_tau."""
    p = int(powers.power)
    if not 1 <= p <= _MAX_POWER:
        raise ValueError(f"ptau: power {p} is out of range (1..{_MAX_POWER})")
    n = 1 << p
    parts = [(sid, getattr(powers, name), count, words) for sid, name, count, words in
             ((2, 'tau_g1', 2 * n - 1, 8), (3, 'tau_g2', n, 16), (4, 'alpha_tau_g1', n, 8), (5, 'beta_tau_g1', n, 8),
              (6, 'beta_g2', 1, 16))]
    lag = powers.lagrange
    if lag is not None:
        if int(lag.power) != p:
            raise ValueError(f"ptau: the Lagrange sections are prepared at power {lag.power}, the ceremony has power {p}")
        parts += [(sid, getattr(lag, name), count, 16 if name == 'tau_g2' else 8)
                  for sid, name, count in zip(_LAGRANGE_IDS, LAGRANGE, lagrange_counts(p))]
    reserve = []
    if points_space:
        reserve = [(sid, count * words * 8) for sid, _, count, words in parts]
        parts = []
    if lag is None and lagrange_space:
        reserve += [(sid, count * (128 if sid == 13 else 64)) for sid, count in zip(_LAGRANGE_IDS, lagrange_counts(p))]
    arrays = []
    for sid, a, count, words in parts:
        a = np.asarray(a)
        if a.dtype.itemsize != 8 or a.ndim != 2 or a.shape != (count, words):
            raise ValueError(f"ptau: section {sid} needs {count} rows of {words} words at power {p}, not shape {a.shape}")
        arrays.append((sid, a))
    own = isinstance(dst, (str, os.PathLike))
    f = open(dst, 'wb') if own else dst
    try:
        f.write(b'ptau' + struct.pack('<II', 1, 1 + len(arrays) + len(reserve)))
        f.write(struct.pack('<IQI', 1, 4 + 32 + 8, 32) + Q_MOD.to_bytes(32, 'little') + struct.pack('<II', p, int(powers.ceremony_power)))
        for sid, a in arrays:
            f.write(struct.pack('<IQ', sid, a.nbytes))
            step = max(1, _WRITE_CHUNK // (a.shape[1] * 8))
            for at in range(0, a.shape[0], step):
                f.write(np.ascontiguousarray(a[at:at + step], dtype='<u8').data)
        for sid, nbytes in reserve:
            f.write(struct.pack('<IQ', sid, nbytes))
            f.seek(nbytes, os.SEEK_CUR)
        if reserve:
            f.truncate()
    finally:
        if own:
            f.close()
