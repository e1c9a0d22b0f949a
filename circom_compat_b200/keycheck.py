"""The verdict of Groth16.verify_proving_key (b2g_setup_check), and the host comparison of a .zkey's coefficient section with
the circuit it claims.

SetupCheck is truthy when the key is the circuit's key on the ceremony; .reason names the first failing check: a count
("h_query holds 4095 points; a CircomReduction domain of 4096 needs 4096"), a field snarkjs copies from the ceremony
("alpha_g1 is not the ceremony's"), a point ("l_query[17]: off the curve", "tau_g2[3]: not in G2"), an equation
("b_g2_query does not match the circuit and ceremony") or the matrices ("matrix A differs from the circuit at row 17").
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .ptau import ARRAYS, _RULES
from .zkey import R_MOD

# b2g_setup_report.field on the key side
KEY_FIELDS = ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'gamma_g2', 'delta_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query',
              'b_g2_query', 'l_query', 'h_query')
G2_FIELDS = ('beta_g2', 'gamma_g2', 'delta_g2', 'b_g2_query', 'tau_g2')
_EQUATIONS = {7: 'a_query does not match the circuit and ceremony', 8: 'b_g1_query does not match the circuit and ceremony',
              9: 'b_g2_query does not match the circuit and ceremony',
              6: 'gamma_abc_g1 / l_query do not match the circuit and ceremony',
              11: 'h_query does not match the circuit and ceremony', 2: 'delta_g1 and delta_g2 disagree'}


@dataclass
class SetupCheck:
    """the verdict of a proving-key check: truthy when the key passes, else .reason says why"""
    ok: bool
    reason: str = None

    def __bool__(self) -> bool:
        return bool(self.ok)


def shape_reason(name: str, have: int, want: int, reduction: str, n: int) -> str:
    if name == 'h_query':
        return f"h_query holds {have} points; a {reduction} domain of {n} needs {want}"
    return f"{name} holds {have} points; the circuit needs {want}"


def report_reason(rep) -> str:
    """the reason of a failed b2g_setup_report"""
    if rep.rule == 8:
        return _EQUATIONS[rep.field]
    name = ARRAYS[rep.field] if rep.side else KEY_FIELDS[rep.field]
    if rep.rule == 6:
        return f"{name}: the circuit needs {rep.index} points"
    if rep.rule == 7:
        return f"{name} is not the ceremony's"
    return f"{name}[{rep.index}]: {_RULES[rep.rule][name in G2_FIELDS]}"


def canonical_rows(mat, m: int) -> list:
    """the rows of a CSR matrix (rowptr, col, Montgomery val) with each row sorted by column, duplicates summed mod r and zeros
    dropped: a list of m tuples of (column, value)"""
    rowptr, col, val = (np.asarray(a) for a in mat)
    raw = np.ascontiguousarray(val, dtype='<u8').tobytes()
    rows = []
    for r in range(m):
        acc = {}
        for k in range(int(rowptr[r]), int(rowptr[r + 1])):
            c = int(col[k])
            acc[c] = (acc.get(c, 0) + int.from_bytes(raw[32 * k:32 * k + 32], 'little')) % R_MOD
        rows.append(tuple(sorted((c, v) for c, v in acc.items() if v)))
    return rows


def matrices_reason(circuit, matrices):
    """None when a .zkey's ConstraintMatrices (read_zkey) hold the circuit's A and B (ConstraintMatrices of the circuit) with
    its counts, else the first difference"""
    for attr, what in (('num_instance_variables', 'num_inputs'), ('num_constraints', 'num_constraints'), ('n_vars', 'n_vars')):
        a, b = getattr(matrices, attr), getattr(circuit, attr)
        if a != b:
            return f"the matrices' {what} {a} differs from the circuit's {b}"
    m = circuit.num_constraints
    for name in ('a', 'b'):
        got, want = canonical_rows(getattr(matrices, name), m), canonical_rows(getattr(circuit, name), m)
        for r in range(m):
            if got[r] != want[r]:
                return f"matrix {name.upper()} differs from the circuit at row {r}"
    return None
