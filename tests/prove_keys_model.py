"""Plain model of the host tables of b2g_pk_group_load / b2g_prove_keys (csrc/prover.cu group_layout, call_layout).

A group of K keys builds each query's tables (H, L, A, B1, B2) into one arena at one window size c, msm_pick_c of the
largest base count of that query in the group; key k's rows of query q start at the sum of nwin(c) x bases over the keys
before it.  A call with counts[k] proofs of key k, key after key, sorts three scalar families:
  H over the call's h vectors (key k's proofs n_dom[k] apart), W over w[1..] (L and A), B over the gathered B scalars
  (B1 and B2); proof j's row of each is (first scalar, first canonical slot, base count, arena row of its key).
"""

QUERIES = ('H', 'L', 'A', 'B1', 'B2')
SORT_QUERY = (0, 2, 3)          # H, A (for L and A), B1 (for B1 and B2)
MAX_BATCH = 65535


class Refused(Exception):
    pass


def pick_c(n):
    """msm.cuh msm_pick_c"""
    if n >= 3 << 18:
        return 17
    if n >= 1 << 19:
        return 16
    if n >= 1 << 15:
        return 15
    if n >= 1 << 13:
        return 13
    if n >= 1 << 11:
        return 11
    return max(8, n.bit_length() - 1 - 3)


def nwin(c):
    return -(-255 // c)


def key_bases(domain, n_vars, b_real=None):
    """a key's base counts per query: b_real = the real B bases of a key whose B query is compacted, else None"""
    nb = n_vars - 1 if b_real is None else b_real
    return (domain, n_vars - 1, n_vars - 1, nb, nb)


def group_layout(bases):
    """bases = [5 base counts per key] -> (c per query, [first arena row per query] per key); Refused at 2^31 rows"""
    if not bases:
        raise Refused('no keys')
    cs = [pick_c(max(b[q] for b in bases) or 1) for q in range(5)]
    rows = [[0] * 5 for _ in bases]
    for q in range(5):
        at = 0
        for k, b in enumerate(bases):
            rows[k][q] = at
            at += b[q] * nwin(cs[q])
            if at >= 1 << 31:
                raise Refused('2^31 rows')
    return cs, rows


def call_layout(cs, rows, bases, n_vars, n_dom, counts):
    """-> three lists (H, W, B sorts) of (src, canon, n, row) per proof; Refused for a total outside [1, MAX_BATCH] or a
    sort reaching 2^32 entries"""
    total = sum(counts)
    if total == 0 or total > MAX_BATCH:
        raise Refused('total count')
    out = [[], [], []]
    tw = tv = 0
    tn = [0, 0, 0]
    for k, cnt in enumerate(counts):
        for _ in range(cnt):
            src = (tv, tw + 1, tn[2])
            for t, q in enumerate(SORT_QUERY):
                out[t].append((src[t], tn[t], bases[k][q], rows[k][q]))
                tn[t] += bases[k][q]
            tw += n_vars[k]
            tv += n_dom[k]
    for t, q in enumerate(SORT_QUERY):
        if tn[t] * nwin(cs[q]) >= 1 << 32 or total << (cs[q] - 1) >= 1 << 32:
            raise Refused('2^32 entries')
    return out
