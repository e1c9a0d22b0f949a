"""ctypes binding of libb2groth.so (include/b2groth.h).  There is NO CPU fallback: if the shared library is missing,
or no CUDA device is present, every entry point raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('B2G_LIB') or os.path.join(_HERE, 'libb2groth.so')   # B2G_LIB: tuning builds only

B2G_OK, B2G_E_DOMAIN, B2G_E_SHAPE, B2G_E_DEVICE, B2G_E_INPUT = 0, -1, -2, -3, -4
PARTIAL_BYTES = 768
IPC_HANDLE_BYTES = 80          # B2G_IPC_HANDLE_BYTES: cudaIpcMemHandle_t + arena capacity
REDUCTION_CIRCOM, REDUCTION_LIBSNARK = 0, 1


class B2gError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b2groth error {code}: {msg}")
        self.code = code
        self.msg = msg


class PolynomialDegreeTooLarge(B2gError):
    """SynthesisError::PolynomialDegreeTooLarge (/root/reference/src/circom/qap.rs:31,66)."""


class PkDesc(C.Structure):
    _fields_ = [('n_vars', C.c_uint32), ('n_public', C.c_uint32), ('domain_size', C.c_uint32), ('reserved', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query',
                                          'b_g2_query', 'l_query', 'h_query')]


class MatDesc(C.Structure):
    _fields_ = [('num_constraints', C.c_uint32), ('num_inputs', C.c_uint32), ('n_vars', C.c_uint32), ('reduction', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('a_rowptr', 'a_col', 'a_val', 'b_rowptr', 'b_col', 'b_val', 'c_rowptr', 'c_col', 'c_val')]


class VkDesc(C.Structure):
    _fields_ = [('n_public', C.c_uint32), ('reserved', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('alpha_g1', 'beta_g2', 'gamma_g2', 'delta_g2', 'gamma_abc_g1')]


class SetupSecrets(C.Structure):
    """b2g_setup_secrets: 32-byte canonical scalars; g1 / g2 affine Montgomery generators or NULL for the standard ones"""
    _fields_ = [(k, C.c_void_p) for k in ('alpha', 'beta', 'gamma', 'delta', 'tau', 'g1', 'g2')]


class SetupOut(C.Structure):
    """b2g_setup_out: host buffers in the b2g_pk_desc layout"""
    _fields_ = [(k, C.c_void_p) for k in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'gamma_g2', 'delta_g2', 'gamma_abc_g1',
                                          'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query')]


class PowersDesc(C.Structure):
    """b2g_powers_desc: the host arrays of a powers-of-tau ceremony of size 2^log_size (affine Montgomery, all-zero = infinity)"""
    _fields_ = [('log_size', C.c_uint32), ('reserved', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')]


class LagrangeDesc(C.Structure):
    """b2g_lagrange_desc / b2g_lagrange_out: the prepared Lagrange sections 12-15 of a ceremony prepared at power log_size"""
    _fields_ = [('log_size', C.c_uint32), ('reserved', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1')]


class PowersReport(C.Structure):
    """b2g_powers_report: the verdict of b2g_powers_check and b2g_lagrange_check (rule 0 ok, 1-5 a point rule, 6 the pairing
    product, 7 a Lagrange section that is not the transform of its powers)"""
    _fields_ = [('ok', C.c_uint8), ('rule', C.c_uint8), ('array', C.c_uint8), ('reserved', C.c_uint8 * 5), ('index', C.c_uint64)]


class PowersSecrets(C.Structure):
    """b2g_powers_secrets: tau, alpha, beta of one phase-1 contribution (32 B canonical each, in [1, r))"""
    _fields_ = [(k, C.c_void_p) for k in ('tau', 'alpha', 'beta')]


class PowersOut(C.Structure):
    """b2g_powers_out: the host arrays b2g_powers_contribute writes, with the counts of its input"""
    _fields_ = [(k, C.c_void_p) for k in ('tau_g1', 'tau_g2', 'alpha_tau_g1', 'beta_tau_g1', 'beta_g2')]


class KeyDesc(C.Structure):
    """b2g_key_desc: a whole proving key with its counts (host arrays)"""
    _fields_ = [(k, C.c_uint32) for k in ('n_vars', 'n_ic', 'n_l', 'n_h')] + \
               [(k, C.c_void_p) for k in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'gamma_g2', 'delta_g2', 'gamma_abc_g1',
                                          'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query')]


class SetupReport(C.Structure):
    """b2g_setup_report: the verdict of b2g_setup_check"""
    _fields_ = [('ok', C.c_uint8), ('rule', C.c_uint8), ('side', C.c_uint8), ('field', C.c_uint8), ('reserved', C.c_uint8 * 4),
                ('index', C.c_uint64)]


class DeltaKey(C.Structure):
    """b2g_delta_key: the fields of a proving key a delta contribution changes (host buffers)"""
    _fields_ = [('n_l', C.c_uint32), ('n_h', C.c_uint32)] + [(k, C.c_void_p) for k in ('delta_g1', 'delta_g2', 'l_query', 'h_query')]


class WasmSummary(C.Structure):
    """b2g_wasm_summary: what b2g_wasm_load read from a circom 2 module"""
    _fields_ = [(k, C.c_uint32) for k in ('n32', 'witness_size', 'input_size', 'version', 'mem_pages')] + \
               [('reserved', C.c_uint32 * 3)]


class WasmLimits(C.Structure):
    """b2g_wasm_limits: per-lane limits of the device interpreter and the device-memory budget of a call"""
    _fields_ = [(k, C.c_uint32) for k in ('max_pages', 'max_depth', 'stack_slots', 'reserved')] + \
               [('fuel', C.c_uint64), ('budget_bytes', C.c_uint64)]


class KeyBatch(C.Structure):
    """b2g_key_batch: one batch of proofs under one verifying key (b2g_verify_batch_keys, b2g_verify_batch_keys_locate)"""
    _fields_ = [('vk', C.c_void_p), ('count', C.c_uint32), ('reserved', C.c_uint32)] + \
               [(k, C.c_void_p) for k in ('public_inputs', 'proofs', 'weights')]


EXPORTS = ['b2g_last_error', 'b2g_version', 'b2g_device_count', 'b2g_ctx_create', 'b2g_ctx_destroy', 'b2g_ctx_prepare', 'b2g_pk_load', 'b2g_pk_free',
           'b2g_matrices_load', 'b2g_matrices_free', 'b2g_witness_map', 'b2g_prove', 'b2g_prove_many', 'b2g_prove_submit', 'b2g_prove_wait', 'b2g_host_register', 'b2g_host_unregister', 'b2g_prove_partial', 'b2g_prove_finish',
           'b2g_p2p_export', 'b2g_p2p_import', 'b2g_p2p_connect_local', 'b2g_prove_sharded_p2p', 'b2g_msm_g1', 'b2g_msm_g2', 'b2g_ntt', 'b2g_fixed_base_g1', 'b2g_fixed_base_g2', 'b2g_test_op', 'b2g_last_timings',
           'b2g_bench_device', 'b2g_bench_msm', 'b2g_launch_count', 'b2g_vk_load', 'b2g_vk_load_many', 'b2g_vk_free', 'b2g_vk_alpha_beta', 'b2g_verify_many',
           'b2g_verify_batch', 'b2g_proofs_decompress', 'b2g_verify_many_compressed', 'b2g_verify_batch_compressed',
           'b2g_verify_batch_locate', 'b2g_verify_batch_locate_compressed', 'b2g_verify_batch_keys',
           'b2g_verify_batch_keys_compressed', 'b2g_verify_batch_keys_locate', 'b2g_verify_batch_keys_locate_compressed',
           'b2g_rerandomize_many', 'b2g_points_serialize', 'b2g_points_deserialize', 'b2g_setup',
           'b2g_setup_from_powers', 'b2g_delta_update', 'b2g_delta_update_check', 'b2g_points_intt',
           'b2g_powers_msm', 'b2g_powers_check', 'b2g_setup_check', 'b2g_powers_prepare', 'b2g_lagrange_check',
           'b2g_setup_from_lagrange', 'b2g_points_scale', 'b2g_powers_contribute',
           'b2g_pk_group_load', 'b2g_pk_group_free', 'b2g_prove_keys', 'b2g_pk_group_layout',
           'b2g_wasm_load', 'b2g_wasm_load_module', 'b2g_wasm_free', 'b2g_wasm_info', 'b2g_wasm_get_limits',
           'b2g_wasm_set_limits', 'b2g_witness_calculate', 'b2g_wasm_run']

_lib = None


def lib():
    """Load libb2groth.so; raises if it has not been built (python __graft_entry__.py / make -C csrc)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `make -C circom_compat_b200/csrc` "
                              "(there is no CPU fallback for the proving path)")
        L = C.CDLL(LIB_PATH)
        L.b2g_last_error.restype = C.c_char_p
        for name in EXPORTS:
            getattr(L, name)  # AttributeError if a declared symbol is not exported
        vp, i, sz = C.c_void_p, C.c_int, C.c_size_t
        L.b2g_ctx_create.argtypes = [i, i, i, C.POINTER(vp)]
        L.b2g_ctx_destroy.argtypes = [vp]
        L.b2g_ctx_prepare.argtypes = [vp, vp, vp]
        L.b2g_pk_load.argtypes = [vp, C.POINTER(PkDesc), C.POINTER(vp)]
        L.b2g_pk_free.argtypes = [vp]
        L.b2g_matrices_load.argtypes = [vp, C.POINTER(MatDesc), C.POINTER(vp)]
        L.b2g_matrices_free.argtypes = [vp]
        L.b2g_witness_map.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_uint32)]
        L.b2g_prove.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.b2g_prove_many.argtypes = [vp, vp, vp, C.c_uint32, vp, vp, vp, vp]
        L.b2g_pk_group_load.argtypes = [vp, C.c_uint32, C.POINTER(PkDesc), vp, C.POINTER(vp)]
        L.b2g_pk_group_free.argtypes = [vp]
        L.b2g_prove_keys.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.b2g_pk_group_layout.argtypes = [C.c_uint32, vp, vp, vp, vp, vp, vp, vp]
        L.b2g_prove_submit.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.b2g_prove_wait.argtypes = [vp]
        L.b2g_host_register.argtypes = [vp, sz]
        L.b2g_host_unregister.argtypes = [vp]
        L.b2g_prove_partial.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.b2g_prove_finish.argtypes = [vp, vp, vp, i, vp, vp, vp]
        L.b2g_p2p_export.argtypes = [vp, vp]
        L.b2g_p2p_import.argtypes = [vp, vp, i]
        L.b2g_p2p_connect_local.argtypes = [vp, i]
        L.b2g_prove_sharded_p2p.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.b2g_msm_g1.argtypes = [vp, vp, vp, sz, i, vp]
        L.b2g_msm_g2.argtypes = [vp, vp, vp, sz, i, vp]
        L.b2g_ntt.argtypes = [vp, vp, i, i]
        L.b2g_fixed_base_g1.argtypes = [vp, vp, sz, vp]
        L.b2g_fixed_base_g2.argtypes = [vp, vp, sz, vp]
        L.b2g_setup.argtypes = [vp, C.POINTER(MatDesc), C.POINTER(SetupSecrets), C.POINTER(SetupOut)]
        L.b2g_setup_from_powers.argtypes = [vp, C.POINTER(MatDesc), C.POINTER(PowersDesc), C.POINTER(SetupOut)]
        L.b2g_delta_update.argtypes = [vp, C.POINTER(DeltaKey), vp, C.POINTER(DeltaKey)]
        L.b2g_delta_update_check.argtypes = [vp, C.POINTER(DeltaKey), C.POINTER(DeltaKey), vp, vp]
        L.b2g_points_intt.argtypes = [vp, i, i, vp]
        L.b2g_powers_msm.argtypes = [vp, i, sz, vp, vp, vp]
        L.b2g_powers_check.argtypes = [vp, C.POINTER(PowersDesc), C.c_uint32, vp, C.POINTER(PowersReport)]
        L.b2g_setup_check.argtypes = [vp, C.POINTER(MatDesc), C.POINTER(PowersDesc), C.POINTER(KeyDesc), vp, C.POINTER(SetupReport)]
        L.b2g_powers_prepare.argtypes = [vp, C.POINTER(PowersDesc), C.POINTER(LagrangeDesc)]
        L.b2g_lagrange_check.argtypes = [vp, C.POINTER(PowersDesc), C.POINTER(LagrangeDesc), C.c_uint32, vp, C.POINTER(PowersReport)]
        L.b2g_setup_from_lagrange.argtypes = [vp, C.POINTER(MatDesc), C.POINTER(PowersDesc), C.POINTER(LagrangeDesc), C.POINTER(SetupOut)]
        L.b2g_points_scale.argtypes = [vp, i, sz, vp, vp, vp]
        L.b2g_powers_contribute.argtypes = [vp, C.POINTER(PowersDesc), C.POINTER(PowersSecrets), C.POINTER(PowersOut)]
        L.b2g_wasm_load.argtypes = [vp, vp, sz, C.POINTER(vp)]
        L.b2g_wasm_load_module.argtypes = [vp, vp, sz, C.POINTER(vp)]
        L.b2g_wasm_free.argtypes = [vp]
        L.b2g_wasm_info.argtypes = [vp, C.POINTER(WasmSummary)]
        L.b2g_wasm_get_limits.argtypes = [vp, C.POINTER(WasmLimits)]
        L.b2g_wasm_set_limits.argtypes = [vp, C.POINTER(WasmLimits)]
        L.b2g_witness_calculate.argtypes = [vp, vp, C.c_uint32, C.c_uint32, vp, vp, vp, i, vp, vp]
        L.b2g_wasm_run.argtypes = [vp, vp, C.c_char_p, C.c_uint32, C.c_uint32, vp, vp, vp]
        L.b2g_test_op.argtypes = [vp, i, vp, vp, sz, vp]
        L.b2g_last_timings.argtypes = [vp, vp]
        L.b2g_bench_device.argtypes = [vp, vp, vp, i, C.POINTER(C.c_float)]
        L.b2g_bench_msm.argtypes = [vp, vp, vp, i, i, C.POINTER(C.c_float)]
        L.b2g_launch_count.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.b2g_device_count.argtypes = [C.POINTER(C.c_int)]
        L.b2g_vk_load.argtypes = [vp, C.POINTER(VkDesc), C.POINTER(vp)]
        L.b2g_vk_load_many.argtypes = [vp, C.c_uint32, C.POINTER(VkDesc), C.POINTER(vp)]
        L.b2g_vk_free.argtypes = [vp]
        L.b2g_vk_alpha_beta.argtypes = [vp, vp]
        L.b2g_verify_many.argtypes = [vp, vp, C.c_uint32, vp, vp, vp]
        L.b2g_verify_batch.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
        L.b2g_proofs_decompress.argtypes = [vp, C.c_uint32, vp, vp, vp]
        L.b2g_verify_many_compressed.argtypes = [vp, vp, C.c_uint32, vp, vp, vp]
        L.b2g_verify_batch_compressed.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
        L.b2g_verify_batch_locate.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
        L.b2g_verify_batch_locate_compressed.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp]
        L.b2g_verify_batch_keys.argtypes = [vp, C.c_uint32, C.POINTER(KeyBatch), vp]
        L.b2g_verify_batch_keys_compressed.argtypes = [vp, C.c_uint32, C.POINTER(KeyBatch), vp]
        L.b2g_verify_batch_keys_locate.argtypes = [vp, C.c_uint32, C.POINTER(KeyBatch), vp]
        L.b2g_verify_batch_keys_locate_compressed.argtypes = [vp, C.c_uint32, C.POINTER(KeyBatch), vp]
        L.b2g_rerandomize_many.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, vp, vp]
        L.b2g_points_serialize.argtypes = [vp, i, i, sz, vp, vp]
        L.b2g_points_deserialize.argtypes = [vp, i, i, sz, vp, vp, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def check(rc: int):
    if rc != B2G_OK:
        msg = lib().b2g_last_error().decode(errors='replace')
        if rc == B2G_E_DOMAIN:
            raise PolynomialDegreeTooLarge(rc, msg)
        raise B2gError(rc, msg)
