"""API-surface mirror of ark-circom's builder (host orchestration only, no compute):

  CircomConfig.new(wtns, r1cs) / CircomBuilder.{new, push_input, setup, build}   <- /root/reference/src/circom/builder.rs:30-117
  CircomCircuit{r1cs, witness}.get_public_inputs()                               <- /root/reference/src/circom/circuit.rs:12-26

`wtns` is the *witness source*:
  - the path of the circuit's circom 2 `.wasm` (recognised by its `\0asm` magic), as CircomConfig::new(wasm, r1cs)
    takes it: build() then computes the witness on the GPU with witness.WitnessCalculator, the device interpreter that
    stands in for the reference's wasmer runtime (src/witness/*);
  - a callable `inputs: dict[str, list[int]] -> list[int]` (e.g. a wrapper around snarkjs);
  - or the path of a `.wtns` file produced for those inputs.
Everything downstream (matrices, setup, prove) is the same as with the reference.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Union

from .r1cs import R1CS, R1CSFile, read_wtns
from .zkey import R_MOD

WitnessSource = Union[str, Callable[[Dict[str, List[int]]], List[int]]]


def _is_wasm(path) -> bool:
    try:
        with open(path, 'rb') as f:
            return f.read(4) == b'\0asm'
    except OSError:              # a .wtns path may name a file that is written later, before build()
        return False


@dataclass
class CircomCircuit:
    r1cs: R1CS
    witness: Optional[List[int]] = None

    def get_public_inputs(self) -> Optional[List[int]]:
        """w[1..num_inputs] (through the wire mapping when one is kept), circuit.rs:18-26"""
        if self.witness is None:
            return None
        if self.r1cs.wire_mapping is None:
            return list(self.witness[1:self.r1cs.num_inputs])
        return [self.witness[i] for i in self.r1cs.wire_mapping[1:self.r1cs.num_inputs]]

    def to_circuit(self):
        """matrices of CircomCircuit::generate_constraints (circuit.rs:30-82) as a synth.Circuit"""
        return self.r1cs.to_circuit()


@dataclass
class CircomConfig:
    r1cs: R1CS
    wtns: WitnessSource
    sanity_check: bool = False
    wasm: Optional[object] = None          # the WitnessCalculator of a .wasm source

    @staticmethod
    def new(wtns: WitnessSource, r1cs_path: str) -> 'CircomConfig':
        with open(r1cs_path, 'rb') as f:
            r1cs = R1CS.from_file(R1CSFile.new(f.read()))
        wasm = None
        if not callable(wtns) and _is_wasm(wtns):
            from .witness import WitnessCalculator
            wasm = WitnessCalculator.new(wtns)
        return CircomConfig(r1cs, wtns, wasm=wasm)


@dataclass
class CircomBuilder:
    cfg: CircomConfig
    inputs: Dict[str, List[int]] = field(default_factory=dict)

    @staticmethod
    def new(cfg: CircomConfig) -> 'CircomBuilder':
        return CircomBuilder(cfg)

    def push_input(self, name: str, val: int) -> None:
        self.inputs.setdefault(str(name), []).append(int(val))

    def setup(self) -> CircomCircuit:
        """circuit without witness, for parameter generation; the wire mapping is disabled (builder.rs:81-82)"""
        r = self.cfg.r1cs
        return CircomCircuit(R1CS(r.num_inputs, r.num_aux, r.num_variables, r.constraints, None), None)

    def build(self) -> CircomCircuit:
        circom = self.setup()
        src = self.cfg.wtns
        if self.cfg.wasm is not None:
            witness = self.cfg.wasm.calculate_witness(self.inputs, self.cfg.sanity_check)
        elif callable(src):
            witness = src(self.inputs)
        else:
            witness = read_wtns(open(src, 'rb').read())
        # negative outputs of a witness calculator map to r - |w| (src/witness/witness_calculator.rs:171-174)
        witness = [int(x) % R_MOD for x in witness]
        if len(witness) != circom.r1cs.num_variables:
            raise ValueError("witness length != number of wires")
        if self.cfg.sanity_check or __debug__:                          # the reference checks satisfiability in debug builds
            for k, (a, b, c) in enumerate(circom.r1cs.constraints):
                ev = [sum(v * witness[i] for i, v in lc) % R_MOD for lc in (a, b, c)]
                if ev[0] * ev[1] % R_MOD != ev[2]:
                    raise ValueError(f"Unsatisfied constraint: {k}")
        circom.witness = witness
        return circom
