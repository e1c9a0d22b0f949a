"""Signed base-2^c digits of MSM scalars.  TEST INFRASTRUCTURE ONLY.

`make_digits` is the full carry-chain decomposition ark-ec 0.5 uses (VariableBaseMSM::msm_bigint).  `digit_at` restates the
device's shortcut (circom_compat_b200/csrc/msm.cu msm_window_bits / msm_digit_at): the carry into window w is found by
walking down only while the windows below hold exactly 2^(c-1) - 1.  `digit_edge_scalars` builds scalars whose windows sit
on the values where that walk decides something: runs of 2^(c-1) - 1 of every depth, windows across a 32-bit limb, r - 1.
"""
from __future__ import annotations

R_MOD = 21888242871839275222246405745257275088548364400416034343698204186575808495617
FR_BITS = 254                     # Fr::MODULUS_BIT_SIZE: the num_bits ark-ec passes to make_digits


def nwin(c: int) -> int:
    """msm.cuh msm_nwin: windows of the device decomposition"""
    return (255 + c - 1) // c


def window_bits(k: int, c: int, w: int) -> int:
    """msm_window_bits: raw c-bit window w of a 256-bit scalar read as 8 x 32-bit limbs"""
    off = w * c
    limb, sh = off >> 5, off & 31
    if limb >= 8:
        return 0
    v = (k >> (32 * limb)) & 0xffffffff
    if limb + 1 < 8 and sh + c > 32:
        v |= ((k >> (32 * (limb + 1))) & 0xffffffff) << 32
    return (v >> sh) & ((1 << c) - 1)


def digit_at(k: int, c: int, w: int) -> int:
    """msm_digit_at: signed digit of window w, the carry found by the walk down through windows equal to 2^(c-1) - 1"""
    half = 1 << (c - 1)
    carry = 0
    for v in range(w - 1, -1, -1):
        b = window_bits(k, c, v)
        if b >= half:
            carry = 1
            break
        if b < half - 1:
            break
    coef = window_bits(k, c, w) + carry
    cout = (coef + half) >> c
    return coef - (cout << c)


def device_digits(k: int, c: int) -> list:
    return [digit_at(k, c, w) for w in range(nwin(c))]


def make_digits(k: int, c: int, num_bits: int = FR_BITS) -> list:
    """ark-ec 0.5 make_digits: one pass from the bottom with the carry; the top digit keeps its carry"""
    radix = 1 << c
    carry = 0
    count = (num_bits + c - 1) // c
    out = []
    for i in range(count):
        coef = carry + ((k >> (i * c)) & (radix - 1))
        carry = (coef + radix // 2) >> c
        d = coef - (carry << c)
        if i == count - 1:
            d += carry << c
        out.append(d)
    return out


def straddling_windows(c: int) -> list:
    """windows that cross a 32-bit limb boundary below bit 254"""
    return [w for w in range(nwin(c)) if (w * c) % 32 + c > 32 and w * c < FR_BITS]


def digit_edge_scalars(c: int, rng) -> list:
    """Scalars k < r whose c-bit windows take values in {0, 1, h-2, h-1, h, h+1, 2^c-1} (h = 2^(c-1)), with
    - runs of h-1 of every depth 1 .. nwin-1 below a window, ended by a window >= h, by one < h-1, or by the bottom;
    - every limb-straddling window at 2^c-1, h and h-1 (and the window below it at h-1);
    - r-1, r-h, 2^(cw) and 2^(cw)-1 for every window w."""
    h = 1 << (c - 1)
    vals = [0, 1, h - 2, h - 1, h, h + 1, (1 << c) - 1]
    nw = nwin(c)
    top_limit = (R_MOD - 1) >> (c * (nw - 1))          # the top window of any k < r holds at most this

    def compose(ws):
        ws = list(ws)
        ws[nw - 1] = min(ws[nw - 1], top_limit)
        k = sum(v << (c * w) for w, v in enumerate(ws))
        if k >= R_MOD:                                  # only the top window can be lowered: runs never reach it
            ws[nw - 1] -= 1
            k = sum(v << (c * w) for w, v in enumerate(ws))
        assert k < R_MOD
        return k

    out = []
    for depth in range(1, nw):
        for t in sorted({depth, nw - 1, rng.randrange(depth, nw)}):   # t receives the carry decided at the end of the run
            lo = t - depth                                            # lowest window of the run
            enders = [None] if lo == 0 else [rng.choice([h, h + 1, (1 << c) - 1]), rng.choice([0, 1, h - 2])]
            for end in enders:
                ws = [rng.choice(vals) for _ in range(nw)]
                for w in range(lo, t):
                    ws[w] = h - 1
                if end is not None:
                    ws[lo - 1] = end
                out.append(compose(ws))
    for w in straddling_windows(c):
        for v in ((1 << c) - 1, h, h - 1):
            ws = [rng.choice(vals) for _ in range(nw)]
            ws[w] = v
            if v == h - 1 and w > 0:
                ws[w - 1] = h - 1
            out.append(compose(ws))
    out += [R_MOD - 1, R_MOD - h]
    for w in range(nw):
        if c * w < FR_BITS:
            out += [1 << (c * w), (1 << (c * w)) - 1]
    assert all(0 <= k < R_MOD for k in out)
    return out


# ---------------------------------------------------------------------------------------------- layouts of the sorted entry list
MSM_BIG_FRAGS = 32          # msm.cuh: a bucket spanning more runs than this is folded by a whole CTA (msm_fold_big_kernel)


def entry_count(k: int, c: int) -> int:
    """entries one scalar contributes to the bucket-sorted list: its non-zero signed digits"""
    return sum(1 for d in make_digits(k, c) if d)


def partial_slab_prefix(sc, c: int) -> int:
    """Length of the longest prefix of the scalars whose entry count is not a multiple of 4.  A G1 CTA's slab of the
    entry list is 128 runs of `chunk` entries, a multiple of 4, so the last CTA's slab is then partial and not a whole
    number of 16-byte units."""
    total = sum(entry_count(k, c) for k in sc)
    for m in range(len(sc), 0, -1):
        if total % 4:
            return m
        total -= entry_count(sc[m - 1], c)
    raise AssertionError('no prefix with a partial slab')


def fold_boundary_scalars(rng, ch: int = 3):
    """Scalars 1, 2, 3, ... (one digit each, in window 0: scalar v lands in bucket v - 1) with bucket sizes chosen so that,
    in runs of `ch` entries, buckets span MSM_BIG_FRAGS and MSM_BIG_FRAGS + 1 runs, each starting on and off a run
    boundary (one-entry filler buckets move the start).  Returns (shuffled scalars, ch)."""
    counts, start = [], 0

    def span(s, cnt):
        return (s + cnt - 1) // ch - s // ch + 1

    for runs, on in ((MSM_BIG_FRAGS, True), (MSM_BIG_FRAGS + 1, True), (MSM_BIG_FRAGS, False), (MSM_BIG_FRAGS + 1, False)):
        if (start % ch == 0) != on:
            fill = ch - start % ch if on else 1
            counts.append(fill)
            start += fill
        assert (start % ch == 0) == on
        cnt = next(k for k in range(1, 4 * ch * runs) if span(start, k) == runs)
        counts.append(cnt)
        start += cnt
    sc = [b + 1 for b, cnt in enumerate(counts) for _ in range(cnt)]
    rng.shuffle(sc)
    return sc, ch
