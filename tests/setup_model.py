"""Big-int model of b2g_setup's device algorithm (circom_compat_b200/csrc/setup.cu), step for step:

    powers      out[k] = scale * x^k                         (ntt_powers)
    Lagrange    L = iNTT_n(1, tau, ..., tau^(n-1))             (ntt_plain, inverse, natural order)
    column sums one product v * L_row per nonzero, the nonzeros sorted by column, summed run by run (radix sort +
                reduce-by-key), the runs scattered into a zeroed vector; a_j += L_(m+j) for the public-input rows
    combination (beta a_j + alpha b_j + c_j) / gamma for j < num_inputs, / delta for the others
    H query     LibsnarkReduction: powers of tau scaled by (tau^n - 1) / delta, n - 1 of them; CircomReduction: the odd entries
                of iNTT_2n(delta^-1 tau^i for i < 2n - 1, then 0)

The tests hold it against the closed forms of synth.setup_scalars and oracle.pyref.trapdoor_setup_scalars."""
from circom_compat_b200.synth import root_of_unity
from circom_compat_b200.zkey import R_MOD


def powers(x: int, count: int, scale: int = 1) -> list:
    out, p = [], scale % R_MOD
    for _ in range(count):
        out.append(p)
        p = p * x % R_MOD
    return out


def intt(values) -> list:
    """inverse radix-2 NTT, natural order in and out: out_i = n^-1 sum_k v_k omega^(-ik)"""
    a = [v % R_MOD for v in values]
    n = len(a)
    j = 0
    for i in range(1, n):                                   # bit-reversal permutation
        bit = n >> 1
        while j & bit:
            j ^= bit
            bit >>= 1
        j |= bit
        if i < j:
            a[i], a[j] = a[j], a[i]
    size = 2
    while size <= n:
        w = pow(root_of_unity(size), -1, R_MOD)
        half = size // 2
        tw = powers(w, half)
        for start in range(0, n, size):
            for k in range(half):
                u, v = a[start + k], a[start + k + half] * tw[k] % R_MOD
                a[start + k], a[start + k + half] = (u + v) % R_MOD, (u - v) % R_MOD
        size <<= 1
    ninv = pow(n, -1, R_MOD)
    return [x * ninv % R_MOD for x in a]


def lagrange(n: int, tau: int) -> list:
    return intt(powers(tau, n))


def column_sums(rows, cols, vals, L, n_vars: int) -> list:
    prods = [(int(c), int(v) * L[int(r)] % R_MOD) for r, c, v in zip(rows, cols, vals)]
    prods.sort(key=lambda e: e[0])                          # stable, like the radix sort
    sums = [0] * n_vars
    k = 0
    while k < len(prods):                                   # one run per column that occurs
        col, acc = prods[k][0], 0
        while k < len(prods) and prods[k][0] == col:
            acc = (acc + prods[k][1]) % R_MOD
            k += 1
        sums[col] = acc
    return sums


def domain_size(m: int, num_inputs: int) -> int:
    n = 1
    while n < m + num_inputs:
        n <<= 1
    return n


def setup_scalars(circ, tau: int, alpha: int, beta: int, gamma: int, delta: int, flavour: str = 'circom') -> dict:
    """every scalar of the key b2g_setup makes for a synth.Circuit: a, b, ic, l, h (and the Lagrange vector)"""
    m, ni, nv = circ.num_constraints, circ.num_inputs, circ.n_vars
    n = domain_size(m, ni)
    L = lagrange(n, tau)
    a, b, c = (column_sums(rows, cols, vals, L, nv) for rows, cols, vals in (circ.A, circ.B, circ.C))
    for j in range(ni):
        a[j] = (a[j] + L[m + j]) % R_MOD
    ginv, dinv = pow(gamma, -1, R_MOD), pow(delta, -1, R_MOD)
    k = [(beta * a[j] + alpha * b[j] + c[j]) * (ginv if j < ni else dinv) % R_MOD for j in range(nv)]
    if flavour == 'libsnark':
        h = powers(tau, n - 1, (pow(tau, n, R_MOD) - 1) * dinv)
    else:
        h = intt(powers(tau, 2 * n - 1, dinv) + [0])[1::2]
    return dict(n=n, lagrange=L, a=a, b=b, ic=k[:ni], l=k[ni:], h=h)
