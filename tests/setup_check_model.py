"""Big-int model of the scalar side of b2g_setup_check (include/b2groth.h): the column weights, the row products c = A'w, Bw,
Cw, their inverse transforms s, and E5's scalars h for each reduction; and the key's scalars (discrete logs) for a known tau,
from the Lagrange coefficients iNTT_n(tau^i), so that tau may lie in the domain."""
from circom_compat_b200 import synth
from circom_compat_b200.zkey import R_MOD
from ptau_model import folded_circom_h, intt


def _entries(mat):
    rows, cols, vals = mat
    return zip([int(r) for r in rows], [int(c) for c in cols], [int(v) % R_MOD for v in vals])


def row_products(circ, w):
    """c^A (with the public-input rows of A'), c^B, c^C over the domain's n rows"""
    n, m = circ.domain_size, circ.num_constraints
    out = []
    for x, mat in enumerate((circ.A, circ.B, circ.C)):
        c = [0] * n
        for r, col, v in _entries(mat):
            c[r] = (c[r] + v * w[col]) % R_MOD
        if x == 0:
            for j in range(circ.num_inputs):
                c[m + j] = (c[m + j] + w[j]) % R_MOD
        out.append(c)
    return out


def scalars(circ, rho, sigma, flavour):
    """(w, v, s^A, s^B, s^C, h): the weights and the ceremony-side scalars of E1-E5"""
    n = circ.domain_size
    w = [pow(rho, j, R_MOD) for j in range(circ.n_vars)]
    v = [pow(sigma, i, R_MOD) for i in range(n if flavour == 'circom' else n - 1)]
    s = [intt(c) for c in row_products(circ, w)]
    h = [0] * (2 * n - 1)
    if flavour == 'circom':
        t = [x * pow(2, -1, R_MOD) % R_MOD for x in intt(v)]
        winv = pow(synth.root_of_unity(2 * n), -1, R_MOD)
        for k in range(n):
            h[k] = t[k] * pow(winv, k, R_MOD) % R_MOD
            if k <= n - 2:
                h[k + n] = (R_MOD - h[k]) % R_MOD
    else:
        for k in range(n - 1):
            h[k] = (R_MOD - v[k]) % R_MOD
            h[k + n] = v[k]
    return (w, v, *s, h)


def key_scalars(circ, tau, alpha, beta, delta, flavour):
    """the discrete logs of a key b2g_setup_from_powers makes and contributions bring to delta (gamma = 1):
    dict of a, b, ic, l, h lists"""
    n, m, ni = circ.domain_size, circ.num_constraints, circ.num_inputs
    L = intt([pow(tau, i, R_MOD) for i in range(n)])
    sums = []
    for x, mat in enumerate((circ.A, circ.B, circ.C)):
        t = [0] * circ.n_vars
        for r, col, v in _entries(mat):
            t[col] = (t[col] + v * L[r]) % R_MOD
        if x == 0:
            for j in range(ni):
                t[j] = (t[j] + L[m + j]) % R_MOD
        sums.append(t)
    a, b, c = sums
    k = [(beta * a[j] + alpha * b[j] + c[j]) % R_MOD for j in range(circ.n_vars)]
    dinv = pow(delta, -1, R_MOD)
    if flavour == 'circom':
        h = [x * dinv % R_MOD for x in folded_circom_h(n, tau)]
    else:
        zt = (pow(tau, n, R_MOD) - 1) * dinv % R_MOD
        h = [pow(tau, i, R_MOD) * zt % R_MOD for i in range(n - 1)]
    return {'a': a, 'b': b, 'ic': k[:ni], 'l': [x * dinv % R_MOD for x in k[ni:]], 'h': h}


def equations(circ, tau, alpha, beta, delta, rho, sigma, flavour, forged=None):
    """E1-E5 in the exponent for a known tau: a list of (name, key side, ceremony side); the pairing equations are divided
    out, e.g. E4's key side is sum w_j IC_j + delta sum w_j L_j.  forged: (name of a scalar vector, index) to perturb"""
    w, v, sa, sb, sc, h = scalars(circ, rho, sigma, flavour)
    vecs = {'sA': sa, 'sB': sb, 'sC': sc, 'h': h}
    if forged:
        name, i = forged
        vecs[name] = list(vecs[name])
        vecs[name][i] = (vecs[name][i] + 1) % R_MOD
    sa, sb, sc, h = vecs['sA'], vecs['sB'], vecs['sC'], vecs['h']
    key = key_scalars(circ, tau, alpha, beta, delta, flavour)
    ni = circ.num_inputs

    def at_tau(s, scale=1):
        return sum(x * pow(tau, k, R_MOD) for k, x in enumerate(s)) * scale % R_MOD

    def weighted(vals, start=0):
        return sum(w[start + j] * x for j, x in enumerate(vals)) % R_MOD

    e4_key = (weighted(key['ic']) + delta * weighted(key['l'], ni)) % R_MOD
    e4_cer = (at_tau(sa, beta) + at_tau(sb, alpha) + at_tau(sc)) % R_MOD
    e5_key = delta * sum(x * y for x, y in zip(v, key['h'])) % R_MOD
    return [('a_query', weighted(key['a']), at_tau(sa)), ('b_g1_query', weighted(key['b']), at_tau(sb)),
            ('b_g2_query', weighted(key['b']), at_tau(sb)), ('gamma_abc_g1 / l_query', e4_key, e4_cer), ('h_query', e5_key, at_tau(h))]
