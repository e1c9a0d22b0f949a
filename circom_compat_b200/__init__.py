"""circom_compat_b200 - H100-native Groth16 (BN254) prover hot path behind the ark-circom API surface.

Host-side mirror of the reference's public interface (/root/reference/src/lib.rs:4-14) for the proving path:
read_zkey, ProvingKey, ConstraintMatrices, CircomReduction, Groth16.  All arithmetic runs in libb2groth.so
(hand-written sm_90a CUDA behind include/b2groth.h); there is no CPU fallback.
"""
from .zkey import read_zkey, ProvingKey, ConstraintMatrices, fr_to_mont, fr_from_mont  # noqa: F401
from .groth16 import Groth16, CircomReduction, LibsnarkReduction, Proof, Context, ProvingKeyGroup, release, release_all  # noqa: F401
from .r1cs import R1CSFile, R1CS, read_wtns  # noqa: F401
from .builder import CircomConfig, CircomBuilder, CircomCircuit  # noqa: F401
from .verifier import VerifyingKey, PreparedVerifyingKey, MalformedVerifyingKey  # noqa: F401
from ._native import B2gError, PolynomialDegreeTooLarge  # noqa: F401
from .ark_serialize import (serialize_proving_key, deserialize_proving_key, serialize_verifying_key,  # noqa: F401
                            deserialize_verifying_key, deserialize_verifying_keys)
from .witness import WitnessCalculator, WitnessError, WasmModule  # noqa: F401
from .ptau import read_ptau, write_ptau, new_powers_of_tau, Lagrange, Powers, PowersCheck  # noqa: F401
