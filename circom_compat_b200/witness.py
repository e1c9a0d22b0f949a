"""circom 2 witness calculation on the GPU: ark-circom's WitnessCalculator (src/witness/witness_calculator.rs) with the
circuit's .wasm run by the library's device interpreter (csrc/wasm.cu, b2g_wasm_load / b2g_witness_calculate).

    calc = WitnessCalculator.new("circuit.wasm")              # or the module's bytes
    w = calc.calculate_witness({"a": [3], "b": [11]})         # one witness, a list of ints
    w_mont, status = calc.calculate_witnesses([{"a": 3, "b": 11}, {"a": 5, "b": 7}])   # many, one lane each

Input values are reduced mod r on the host, negative values to r - |v| as snarkjs does, and each input name is hashed
(FNV-1a 64) on the host.  A lane that calls the circuit's exceptionHandler stops there and reports the exception; the
reference's runtime ignores that call and keeps computing.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, List, Sequence, Tuple, Union

import numpy as np

from . import _native as N
from .zkey import R_MOD

Inputs = Union[Dict[str, Union[int, Sequence[int]]], Iterable[Tuple[str, Union[int, Sequence[int]]]]]

OK, UNREACHABLE, MEMORY, DIV_ZERO, OVERFLOW, STACK, FUEL, INDIRECT, PROTOCOL = range(9)
EXCEPTION = 0x100
_TRAPS = {UNREACHABLE: "unreachable executed", MEMORY: "memory access out of bounds", DIV_ZERO: "integer divide by zero",
          OVERFLOW: "integer overflow", STACK: "call stack exhausted", FUEL: "instruction budget (fuel) exhausted",
          INDIRECT: "bad call_indirect", PROTOCOL: "getWitnessSize disagrees with the module's witness size"}
# the codes circom 2 passes to runtime.exceptionHandler
_EXCEPTIONS = {1: "Signal not found", 2: "Too many signals set", 3: "Signal already set", 4: "Assert Failed",
               5: "Not enough memory", 6: "Input signal array access exceeds the size"}


def status_name(status: int) -> str:
    if status == OK:
        return "ok"
    if status >= EXCEPTION:
        code = status - EXCEPTION
        return _EXCEPTIONS.get(code, f"Unknown error (exception code {code})")
    return _TRAPS.get(status, f"status {status}")


class WitnessError(RuntimeError):
    """a witness could not be computed: .status is the lane status, str() names the circom exception or the trap"""

    def __init__(self, status: int, index: int = 0):
        super().__init__(f"witness {index}: {status_name(status)}")
        self.status, self.index = status, index


def fnv(name: str) -> Tuple[int, int]:
    """(msb, lsb) of the FNV-1a 64-bit hash of an input name, as setInputSignal takes it"""
    h = 0xcbf29ce484222325
    for b in name.encode():
        h = ((h ^ b) * 0x100000001b3) & 0xffffffffffffffff
    return h >> 32, h & 0xffffffff


def _normalise(inputs: Inputs) -> List[Tuple[str, List[int]]]:
    items = inputs.items() if isinstance(inputs, dict) else inputs
    out = []
    for name, v in items:
        vals = [v] if isinstance(v, (int, np.integer, str)) else list(v)
        out.append((str(name), [int(x) % R_MOD for x in vals]))
    return out


def _ctx(ctx):
    if ctx is None:
        from .groth16 import default_context
        ctx = default_context()
    return ctx


class WasmModule:
    """any module of the interpreter's integer subset (b2g_wasm_load_module), for calling its exports lane by lane"""

    def __init__(self, data: bytes, ctx=None, _circom: bool = False):
        self.ctx = _ctx(ctx)
        self._data = bytes(data)
        self._h = C.c_void_p()
        fn = N.lib().b2g_wasm_load if _circom else N.lib().b2g_wasm_load_module
        N.check(fn(self.ctx._h, self._data, len(self._data), C.byref(self._h)))

    def close(self):
        if getattr(self, '_h', None):
            N.lib().b2g_wasm_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def limits(self) -> N.WasmLimits:
        lim = N.WasmLimits()
        N.check(N.lib().b2g_wasm_get_limits(self._h, C.byref(lim)))
        return lim

    def set_limits(self, max_pages=None, max_depth=None, stack_slots=None, fuel=None, budget_bytes=None):
        """changes the per-lane limits and the device-memory budget; None keeps a value"""
        lim = self.limits
        for k, v in (('max_pages', max_pages), ('max_depth', max_depth), ('stack_slots', stack_slots), ('fuel', fuel),
                     ('budget_bytes', budget_bytes)):
            if v is not None:
                setattr(lim, k, int(v))
        N.check(N.lib().b2g_wasm_set_limits(self._h, C.byref(lim)))

    def run(self, name: str, args) -> Tuple[np.ndarray, np.ndarray]:
        """one lane per row of args (count x nargs integers): (results uint64, status uint32), one per lane"""
        a = np.ascontiguousarray(np.asarray(args, dtype=np.uint64).reshape(len(args), -1))
        count, nargs = a.shape
        res = np.zeros(count, dtype=np.uint64)
        st = np.zeros(count, dtype=np.uint32)
        N.check(N.lib().b2g_wasm_run(self.ctx._h, self._h, name.encode(), count, nargs,
                                     C.c_void_p(a.ctypes.data) if a.size else None, C.c_void_p(res.ctypes.data),
                                     C.c_void_p(st.ctypes.data)))
        return res, st


class WitnessCalculator(WasmModule):
    """a circom 2 circuit's witness calculator on the GPU (WitnessCalculator::new, witness_calculator.rs)"""

    def __init__(self, data: bytes, ctx=None):
        super().__init__(data, ctx, _circom=True)
        info = N.WasmSummary()
        N.check(N.lib().b2g_wasm_info(self._h, C.byref(info)))
        self.n32, self.witness_size, self.input_size = info.n32, info.witness_size, info.input_size
        self.version = info.version
        self.prime = R_MOD                               # b2g_wasm_load refuses any other prime
        self.n64 = ((self.prime.bit_length() - 1) // 64) + 1

    @staticmethod
    def new(path_or_bytes, ctx=None) -> 'WitnessCalculator':
        if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
            return WitnessCalculator(bytes(path_or_bytes), ctx)
        with open(path_or_bytes, 'rb') as f:
            return WitnessCalculator(f.read(), ctx)

    def calculate_witnesses(self, inputs: Sequence[Inputs], sanity_check: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """many witnesses in one call, one device lane each.  Every element of `inputs` names the same inputs with the
        same number of values.  Returns (w_mont, status): w_mont is count x (witness_size * 4) uint64, Montgomery
        form, the rows Groth16.create_proofs accepts (all zeros where status is not 0); status holds one lane status
        per witness (0 ok, see status_name)."""
        norm = [_normalise(i) for i in inputs]
        count = len(norm)
        n = self.witness_size
        if count == 0:
            return np.zeros((0, 4 * n), dtype=np.uint64), np.zeros(0, dtype=np.uint32)
        shape = [(nm, len(v)) for nm, v in norm[0]]
        for k, i in enumerate(norm):
            if [(nm, len(v)) for nm, v in i] != shape:
                raise ValueError(f"calculate_witnesses: inputs[{k}] does not have the names and lengths of inputs[0]")
        hashes = np.array([(lambda m, l: (m << 32) | l)(*fnv(nm)) for nm, _ in shape], dtype=np.uint64)
        counts = np.array([c for _, c in shape], dtype=np.uint32)
        buf = b''.join(v.to_bytes(32, 'little') for i in norm for _, vs in i for v in vs)
        vals = np.frombuffer(buf, dtype=np.uint8) if buf else np.zeros(0, dtype=np.uint8)
        w = np.zeros((count, 4 * n), dtype=np.uint64)
        st = np.zeros(count, dtype=np.uint32)
        p = lambda a: C.c_void_p(a.ctypes.data) if a.size else None   # noqa: E731
        N.check(N.lib().b2g_witness_calculate(self.ctx._h, self._h, count, len(shape), p(hashes), p(counts), p(vals),
                                              int(bool(sanity_check)), p(w), p(st)))
        return w, st

    def calculate_witness(self, inputs: Inputs, sanity_check: bool = False) -> List[int]:
        """calculate_witness: the witness as a list of ints; raises WitnessError on a circom exception or a trap"""
        from .zkey import fr_from_mont
        w, st = self.calculate_witnesses([inputs], sanity_check)
        if st[0]:
            raise WitnessError(int(st[0]))
        return fr_from_mont(w[0])

    def calculate_witness_element(self, inputs: Inputs, sanity_check: bool = False) -> List[int]:
        """calculate_witness_element: the witness as field elements of Fr (ints in [0, r))"""
        return [int(x) % R_MOD for x in self.calculate_witness(inputs, sanity_check)]
