"""Host-side mirror of the proving entry points ark-circom users call, running on libb2groth.so.

    Groth16.create_proof_with_reduction_and_matrices(pk, r, s, matrices, num_inputs, num_constraints, full_assignment)
        <- Groth16::<Bn254, CircomReduction>::create_proof_with_reduction_and_matrices
           (/root/reference/src/zkey.rs:903-912, benches/groth16.rs:52-61)
    CircomReduction.witness_map_from_matrices(matrices, num_inputs, num_constraints, full_assignment)
        <- /root/reference/src/circom/qap.rs:23-88
    Groth16.prove(pk, matrices, full_assignment, rng)
        <- Groth16::<Bn254, CircomReduction>::prove (src/zkey.rs:866): draws r then s, then the call above.
    Groth16.create_proofs(pk, rs, matrices, assignments)
        <- the first call above for many witnesses of one circuit, proved together in one device pass (b2g_prove_many).
    Groth16.load_proving_keys([(pk, matrices), ...]) / Groth16.create_proofs_keys(group, [(rs, assignments), ...])
        <- create_proofs for batches of witnesses under many keys, proved together in one device pass (b2g_prove_keys).
    Groth16.verify_many(vk, public_inputs, proofs)
        <- Groth16::verify_with_processed_vk (src/zkey.rs:869-870, 914-916) for many proofs of one key in one device pass
           (b2g_verify_many, with the key prepared on the device by b2g_vk_load <- process_vk).
    Groth16.verify_batch(vk, public_inputs, proofs)
        <- the same check for a whole batch at once: one random-linear-combination pairing check (b2g_verify_batch).
    Groth16.verify_batch_locate(vk, public_inputs, proofs)
        <- verify_with_processed_vk for every proof, from one batch check per group of 64 proofs (b2g_verify_batch_locate).
    Groth16.load_verifying_keys(vks)
        <- process_vk for many keys in one device pass (b2g_vk_load_many); the keyed verifiers below load their new keys so.
    Groth16.verify_batch_keys([(vk, public_inputs, proofs), ...])
        <- verify_batch for many keys in one device pass, one verdict per key (b2g_verify_batch_keys).
    Groth16.verify_batch_keys_locate([(vk, public_inputs, proofs), ...])
        <- verify_batch_locate for many keys in one device pass, one verdict per proof (b2g_verify_batch_keys_locate).
    Groth16.decompress_proofs(blobs)
        <- Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5, Validate::Yes) for many 128-byte proofs, on the device.
    Groth16.verify_many_compressed / verify_batch_compressed(vk, public_inputs, blobs)
        <- deserialize_compressed followed by verify_many / verify_batch, decoded on the device.
    Groth16.rerandomize_proof(vk, proof, rng) / Groth16.rerandomize_proofs(vk, proofs)
        <- Groth16::rerandomize_proof (ark-groth16 0.5.0), for one or many proofs of one key in one device pass.
    Groth16.generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, g1, g2, tau=tau)
        <- Groth16::generate_parameters_with_qap (ark-groth16 0.5): the whole setup on the device (b2g_setup);
           generate_random_parameters_with_reduction(circuit, rng) draws the toxic waste and calls it.
    Groth16.generate_parameters_from_powers_of_tau(circuit, powers)
        <- snarkjs groth16 setup: a key from a powers-of-tau ceremony (ptau.read_ptau), gamma = delta = 1.
    Groth16.contribute(pk) / Groth16.verify_contribution(before, after)
        <- snarkjs zkey contribute / the delta checks of snarkjs zkey verify.
    Groth16.verify_proving_key(circuit, powers, pk, matrices)
        <- snarkjs zkey verify circuit.r1cs pot.ptau circuit.zkey: the key against its circuit and ceremony (b2g_setup_check).
Arguments keep the reference's meaning; field elements are (n, 4) uint64 Montgomery limb arrays (fr_to_mont).
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .zkey import ConstraintMatrices, ProvingKey, R_MOD


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else C.c_void_p(0)


def _c(a, dtype=np.uint64):
    return np.ascontiguousarray(a, dtype=dtype)


# b2g_test_op (include/b2groth.h): 64-bit words per row of operand a, operand b (0: not read) and the result
_TEST_OP_WORDS = {**{op: (4, 4, 4) for op in (0, 1, 2, 3, 4, 5, 14, 15, 16)}, 6: (4, 0, 4), 7: (4, 0, 4),
                  8: (8, 8, 8), 10: (8, 0, 8), 12: (8, 8, 8), 9: (16, 16, 16), 11: (16, 0, 16), 13: (16, 16, 16),
                  17: (8, 8, 8), 18: (8, 8, 8), 19: (8, 8, 8), 28: (8, 8, 8),
                  20: (16, 16, 16), 21: (16, 8, 16), 22: (16, 0, 16), 23: (32, 32, 32), 24: (32, 16, 32), 25: (32, 0, 32),
                  26: (32, 20, 32), 27: (16 * 20, 0, 32), 29: (4, 4, 8),
                  # the pairing tower (csrc/pairing.cuh): Fq12 = 48 words, G1 / G2 affine = 8 / 16, a line (3 Fq2) = 24
                  30: (48, 48, 48), **{op: (48, 0, 48) for op in (31, 32, 33, 34, 35, 36, 38)}, 37: (8, 16, 48), 39: (48, 24, 48),
                  40: (8, 16, 48), 41: (24, 0, 48), 42: (24, 16, 48),
                  # the batch check's pieces: G2 membership, 128-bit G1 product, cyclotomic exponentiation
                  43: (16, 0, 1), 44: (8, 2, 8), 45: (48, 4, 48),
                  # the compressed-proof decoder's pieces: Fq and Fq2 square roots, one compressed G2 point (result, then a flag slot)
                  46: (4, 0, 8), 47: (8, 0, 12), 48: (8, 0, 20),
                  # the verifier's stages: a verify_many Miller value, prepared lines, the window-table product (b: one
                  # G1 point for every row), the window table and verify_batch's prepared-pair Miller value
                  49: (72, 0, 48), 50: (16, 0, 88 * 24), 51: (4, 8, 16), 52: (8, 0, 32 * 255 * 8), 53: (64, 0, 48),
                  54: (4, 0, 16)}
_TEST_OP_B_ONCE = {51}        # ops whose operand b is one row for all rows of a
TEST_PAIR_RUN = 16            # entries per row of op 27; an entry is 16 words of affine point + 4 words whose bit 0 is the sign


# Device-resident keys / matrices are cached per (host object, device, shard): every Context of that device and shard
# can use them, so several proofs can be in flight on one GPU (one Context per in-flight proof) without duplicating
# the 6 GiB of tables.  Device verifying keys (b2g_vk_load) are cached the same way per (host key object, device).
# release(obj) / release_all() free them.
_PK_HANDLES, _MAT_HANDLES, _VK_HANDLES = {}, {}, {}
_CACHES = ((_PK_HANDLES, 'b2g_pk_free'), (_MAT_HANDLES, 'b2g_matrices_free'), (_VK_HANDLES, 'b2g_vk_free'))


def _vk_desc(key):
    """(b2g_vk_desc, the arrays it points into) of a verifier.VerifyingKey, PreparedVerifyingKey or ProvingKey"""
    from . import verifier
    vk = key.vk if isinstance(key, verifier.PreparedVerifyingKey) else key
    if not isinstance(vk, verifier.VerifyingKey):
        vk = verifier.VerifyingKey.from_proving_key(vk)
    keep = {'alpha_g1': _mont_points([vk.alpha_g1], False), 'beta_g2': _mont_points([vk.beta_g2], True),
            'gamma_g2': _mont_points([vk.gamma_g2], True), 'delta_g2': _mont_points([vk.delta_g2], True),
            'gamma_abc_g1': _mont_points(vk.gamma_abc_g1, False)}
    d = N.VkDesc()
    d.n_public = len(vk.gamma_abc_g1) - 1
    for name, arr in keep.items():
        setattr(d, name, arr.ctypes.data)
    return d, keep


def _mat_desc(m: ConstraintMatrices, n_vars: int, reduction: int, with_c: bool = False):
    """(b2g_mat_desc, the arrays it points into) of ConstraintMatrices; with_c: pass the C matrix whatever the reduction
    (b2g_setup reads it for both)"""
    d = N.MatDesc()
    d.num_constraints, d.num_inputs, d.n_vars, d.reduction = m.num_constraints, m.num_instance_variables, n_vars, reduction
    keep = [_c(m.a[0], np.uint32), _c(m.a[1], np.uint32), _c(m.a[2]), _c(m.b[0], np.uint32), _c(m.b[1], np.uint32), _c(m.b[2])]
    names = ['a_rowptr', 'a_col', 'a_val', 'b_rowptr', 'b_col', 'b_val']
    if with_c or reduction == N.REDUCTION_LIBSNARK:
        if m.c is None:
            raise ValueError(("the setup" if with_c else "LibsnarkReduction") + " needs the C matrix (R1CS route); zkey matrices have none")
        keep += [_c(m.c[0], np.uint32), _c(m.c[1], np.uint32), _c(m.c[2])]
        names += ['c_rowptr', 'c_col', 'c_val']
    for name, arr in zip(names, keep):
        setattr(d, name, arr.ctypes.data if arr.size else None)
    return d, keep


_LOAD_MANY_KEY = re.compile(r'b2g_vk_load_many: key (\d+): (.*)', re.S)


def _refused_key(e):
    """(the key's index in the call, the message b2g_vk_load gives for that key alone) of a b2g_vk_load_many error that names
    a key, else (None, the message)"""
    m = _LOAD_MANY_KEY.fullmatch(e.msg)
    return (int(m.group(1)), m.group(2)) if m else (None, e.msg)


def release(obj):
    if isinstance(obj, ProvingKeyGroup):
        obj._free()
        return
    for cache, free in _CACHES:
        for key in [k for k in cache if k[0] == id(obj)]:
            getattr(N.lib(), free)(cache.pop(key)[0])


def release_all():
    for cache, free in _CACHES:
        for key in list(cache):
            getattr(N.lib(), free)(cache.pop(key)[0])


class ProvingKeyGroup:
    """K proving keys loaded on one device for proving under all of them in one pass (Groth16.load_proving_keys,
    b2g_pk_group_load).  It owns its device state and the matrix handles of its keys; release(group) frees them."""

    def __init__(self, device: int, keys: list, h, mat_handles: list):
        self.device, self.keys, self._h, self._mats = device, keys, h, mat_handles

    @property
    def n_keys(self) -> int:
        return len(self.keys)

    def _free(self):
        if self._h:
            N.lib().b2g_pk_group_free(self._h)
            self._h = C.c_void_p()
        for h in self._mats:
            N.lib().b2g_matrices_free(h)
        self._mats = []

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass


def _pk_desc(pk: ProvingKey):
    """(b2g_pk_desc, the arrays it points into) of a ProvingKey"""
    d = N.PkDesc()
    d.n_vars, d.n_public, d.domain_size = pk.n_vars, pk.n_public, pk.domain_size
    keep = {}
    for name in ('alpha_g1', 'beta_g1', 'delta_g1', 'beta_g2', 'delta_g2', 'a_query', 'b_g1_query', 'b_g2_query', 'l_query', 'h_query'):
        keep[name] = _c(getattr(pk, name))
        setattr(d, name, keep[name].ctypes.data if keep[name].size else None)
    return d, keep


class Context:
    """One b2g_ctx = one in-flight proof on one GPU (optionally one shard of a base-range-sharded prover)."""

    def __init__(self, device: int = 0, shard_rank: int = 0, shard_count: int = 1):
        self._h = C.c_void_p()
        N.check(N.lib().b2g_ctx_create(device, shard_rank, shard_count, C.byref(self._h)))
        self.device, self.shard_rank, self.shard_count = device, shard_rank, shard_count

    def close(self):
        if self._h:
            N.lib().b2g_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def pk_handle(self, pk: ProvingKey):
        key = (id(pk), self.device, self.shard_rank, self.shard_count)
        if key not in _PK_HANDLES:
            d, keep = _pk_desc(pk)
            h = C.c_void_p()
            N.check(N.lib().b2g_pk_load(self._h, C.byref(d), C.byref(h)))
            _PK_HANDLES[key] = (h, pk)
        return _PK_HANDLES[key][0]

    def mat_handle(self, m: ConstraintMatrices, n_vars: int, reduction: int = N.REDUCTION_CIRCOM):
        key = (id(m), self.device, n_vars, reduction)
        if key not in _MAT_HANDLES:
            d, keep = _mat_desc(m, n_vars, reduction)
            h = C.c_void_p()
            N.check(N.lib().b2g_matrices_load(self._h, C.byref(d), C.byref(h)))
            _MAT_HANDLES[key] = (h, m)
        return _MAT_HANDLES[key][0]

    def vk_handle(self, key):
        """device verifying key for a verifier.VerifyingKey, PreparedVerifyingKey or ProvingKey (cached per host object)"""
        cache_key = (id(key), self.device)
        if cache_key not in _VK_HANDLES:
            d, keep = _vk_desc(key)
            h = C.c_void_p()
            N.check(N.lib().b2g_vk_load(self._h, C.byref(d), C.byref(h)))
            _VK_HANDLES[cache_key] = (h, key)
        return _VK_HANDLES[cache_key][0]

    def vk_handles(self, keys) -> list:
        """device verifying keys for many keys, each as vk_handle takes it: every key not yet cached on this device is loaded
        in ONE b2g_vk_load_many call and cached as vk_handle caches it.  Returns the handles in the order of `keys`.  A key
        the library refuses raises B2gError naming its first index in `keys`; then no key of the call is loaded."""
        keys = list(keys)
        loads, at = {}, []
        for i, key in enumerate(keys):
            cache_key = (id(key), self.device)
            if cache_key not in _VK_HANDLES and cache_key not in loads:
                loads[cache_key] = (key,) + _vk_desc(key)
                at.append(i)
        try:
            self._vk_load_many(list(loads.values()))
        except N.B2gError as e:
            i, msg = _refused_key(e)
            raise N.B2gError(e.code, msg if i is None else f"key {at[i]}: {msg}") from e
        return [_VK_HANDLES[(id(key), self.device)][0] for key in keys]

    def _vk_load_many(self, loads):
        """loads = [(key, b2g_vk_desc, the arrays it points into)] of keys not cached on this device: one b2g_vk_load_many
        call, then each handle cached as vk_handle caches it"""
        if not loads:
            return
        descs = (N.VkDesc * len(loads))(*[d for _, d, _ in loads])
        hs = (C.c_void_p * len(loads))()
        N.check(N.lib().b2g_vk_load_many(self._h, len(loads), descs, hs))
        for (key, _, _), h in zip(loads, hs):
            _VK_HANDLES[(id(key), self.device)] = (C.c_void_p(h), key)

    def prepare(self, pk: ProvingKey, matrices: ConstraintMatrices, reduction_id: int = N.REDUCTION_CIRCOM) -> None:
        """load (pk, matrices) and allocate this context's scratch now instead of inside the first proof"""
        N.check(N.lib().b2g_ctx_prepare(self._h, self.pk_handle(pk), self.mat_handle(matrices, pk.n_vars, reduction_id)))

    def p2p_export(self) -> bytes:
        buf = np.zeros(N.IPC_HANDLE_BYTES, dtype=np.uint8)
        N.check(N.lib().b2g_p2p_export(self._h, _ptr(buf)))
        return buf.tobytes()

    def p2p_import(self, handles) -> None:
        blob = np.frombuffer(b''.join(handles), dtype=np.uint8).copy()
        N.check(N.lib().b2g_p2p_import(self._h, _ptr(blob), len(handles)))

    def last_timings(self) -> dict:
        buf = (C.c_float * 16)()
        N.check(N.lib().b2g_last_timings(self._h, buf))
        names = ('h2d', 'witness_map', 'msm_h', 'msm_l', 'msm_a', 'msm_b1', 'msm_b2', 'glue_d2h', 'total', 'host_upload_enqueued', 'host_all_enqueued', 'host_wait')
        return dict(zip(names, list(buf)[:12]))

    def bench_device(self, pk, matrices, iters: int) -> float:
        """average CUDA-event ms of witness map + 5 MSMs + glue with the witness already resident in HBM"""
        ms = C.c_float()
        N.check(N.lib().b2g_bench_device(self._h, self.pk_handle(pk), self.mat_handle(matrices, pk.n_vars), iters, C.byref(ms)))
        return ms.value

    def bench_msm(self, pk, matrices, query: int, iters: int):
        """(whole-MSM ms, accumulate-kernel ms) for one query run alone: 0 H, 1 L, 2 A, 3 B1, 4 B2"""
        out = (C.c_float * 2)()
        N.check(N.lib().b2g_bench_msm(self._h, self.pk_handle(pk), self.mat_handle(matrices, pk.n_vars), query, iters, out))
        return out[0], out[1]

    def launch_count(self) -> int:
        v = C.c_uint64()
        N.check(N.lib().b2g_launch_count(self._h, C.byref(v)))
        return v.value

    # kernel-level entry points -------------------------------------------------------------
    def msm_g1(self, bases, scalars, scalars_mont=False) -> np.ndarray:
        bases, scalars = _c(bases), _c(scalars)
        n = min(bases.size // 8, scalars.size // 4)
        out = np.zeros(8, dtype=np.uint64)
        N.check(N.lib().b2g_msm_g1(self._h, _ptr(bases), _ptr(scalars), n, int(scalars_mont), _ptr(out)))
        return out

    def msm_g2(self, bases, scalars, scalars_mont=False) -> np.ndarray:
        bases, scalars = _c(bases), _c(scalars)
        n = min(bases.size // 16, scalars.size // 4)
        out = np.zeros(16, dtype=np.uint64)
        N.check(N.lib().b2g_msm_g2(self._h, _ptr(bases), _ptr(scalars), n, int(scalars_mont), _ptr(out)))
        return out

    def ntt(self, data_mont, inverse=False) -> np.ndarray:
        d = _c(data_mont).copy()
        n = d.size // 4
        log_n = n.bit_length() - 1
        if n == 0 or (1 << log_n) != n:
            raise ValueError("ntt length must be a power of two")
        N.check(N.lib().b2g_ntt(self._h, _ptr(d), log_n, int(inverse)))
        return d

    def points_intt(self, points_mont, g2=False) -> np.ndarray:
        """b2g_points_intt: the inverse transform (scaled by n^-1) of 2^k affine Montgomery points, rows of 8 / 16 words"""
        d = _c(points_mont).reshape(-1, 16 if g2 else 8).copy()
        n = d.shape[0]
        log_n = n.bit_length() - 1
        if n == 0 or (1 << log_n) != n:
            raise ValueError("points_intt length must be a power of two")
        N.check(N.lib().b2g_points_intt(self._h, int(bool(g2)), log_n, _ptr(d)))
        return d

    def powers_msm(self, points, rho, g2=False) -> np.ndarray:
        """b2g_powers_msm: sum_i rho^i P_i over affine Montgomery points (rows of 8 / 16 words, read in place when contiguous)
        and an int rho in [0, r), as the tableless streamed MSM of verify_powers_of_tau computes it; affine, 8 / 16 words"""
        pts = _c(points).reshape(-1, 16 if g2 else 8)
        rho = int(rho)
        if not 0 <= rho < 1 << 256:
            raise ValueError("rho must be a 256-bit unsigned integer")
        rb = np.frombuffer(rho.to_bytes(32, 'little'), dtype=np.uint8).copy()
        out = np.zeros(16 if g2 else 8, dtype=np.uint64)
        N.check(N.lib().b2g_powers_msm(self._h, int(bool(g2)), pts.shape[0], _ptr(pts), _ptr(rb), _ptr(out)))
        return out

    def points_scale(self, points, scalars, g2=False) -> np.ndarray:
        """b2g_points_scale: k_i P_i for affine Montgomery points (rows of 8 / 16 words) and one canonical scalar per point (ints
        in [0, r), or rows of 4 uint64 words); affine rows of 8 / 16 words.  G2 points must be in G2: they are not checked."""
        pts = _c(points).reshape(-1, 16 if g2 else 8)
        if isinstance(scalars, np.ndarray):
            sc = _c(scalars).reshape(-1, 4)
        else:
            sc = np.frombuffer(b''.join(int(k).to_bytes(32, 'little') for k in scalars), dtype='<u8').reshape(-1, 4)
        if sc.shape[0] != pts.shape[0]:
            raise ValueError(f"points_scale: {pts.shape[0]} points and {sc.shape[0]} scalars")
        out = np.zeros_like(pts)
        N.check(N.lib().b2g_points_scale(self._h, int(bool(g2)), pts.shape[0], _ptr(pts), _ptr(sc), _ptr(out)))
        return out

    def fixed_base_g1(self, scalars_canon) -> np.ndarray:
        sc = _c(scalars_canon); n = sc.size // 4
        out = np.zeros((n, 8), dtype=np.uint64)
        N.check(N.lib().b2g_fixed_base_g1(self._h, _ptr(sc), n, _ptr(out)))
        return out

    def fixed_base_g2(self, scalars_canon) -> np.ndarray:
        sc = _c(scalars_canon); n = sc.size // 4
        out = np.zeros((n, 16), dtype=np.uint64)
        N.check(N.lib().b2g_fixed_base_g2(self._h, _ptr(sc), n, _ptr(out)))
        return out

    def test_op(self, op: int, a, b=None) -> np.ndarray:
        """b2g_test_op: n rows of operand a (and b), returns (n, result words) uint64.  Sizes per op: _TEST_OP_WORDS."""
        a = _c(a); b = _c(b) if b is not None else None
        a_words, b_words, out_words = _TEST_OP_WORDS.get(op, (4, 4, 4))    # an unknown op is refused by the library
        n = a.size // a_words
        b_rows = 1 if op in _TEST_OP_B_ONCE else n
        if b is not None and b_words and b.size < b_rows * b_words:
            raise ValueError(f"test op {op}: operand b holds fewer than {b_rows} rows of {b_words} words")
        out = np.zeros((n, out_words), dtype=np.uint64)
        N.check(N.lib().b2g_test_op(self._h, op, _ptr(a), _ptr(b) if b is not None else None, n, _ptr(out)))
        return out


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


@dataclass
class Proof:
    """Proof<Bn254>{a: G1Affine, b: G2Affine, c: G1Affine}; `data` is the 256-byte uncompressed canonical view."""
    data: bytes

    def _int(self, i):
        return int.from_bytes(self.data[32 * i:32 * i + 32], 'little')

    @property
    def a(self):
        return (self._int(0), self._int(1))

    @property
    def b(self):
        return ((self._int(2), self._int(3)), (self._int(4), self._int(5)))

    @property
    def c(self):
        return (self._int(6), self._int(7))


class PendingProof:
    """A proof submitted with Groth16.submit; keeps the witness and output buffers alive until wait()."""

    def __init__(self, ctx, out, w):
        self._ctx, self._out, self._w = ctx, out, w

    def wait(self) -> Proof:
        N.check(N.lib().b2g_prove_wait(self._ctx._h))
        self._w = None
        return Proof(self._out.tobytes())


COMPRESSED_PROOF_BYTES = 128


def _proof_rows(fn, proofs, compressed) -> bytes:
    """proofs as back-to-back rows: 256-byte Proof.data, or (compressed) 128-byte blobs of any other length refused"""
    if not compressed:
        return b''.join(p.data for p in proofs)
    for b in proofs:
        if not isinstance(b, (bytes, bytearray, memoryview)) or len(b) != COMPRESSED_PROOF_BYTES:
            raise ValueError(f"{fn}: a compressed proof is {COMPRESSED_PROOF_BYTES} bytes")
    return b''.join(bytes(b) for b in proofs)


def _verify_args(fn, vk, public_inputs, proofs, ctx, compressed=False):
    """the argument checks and encoding the verifiers share: None for an empty batch, else (ctx, device key, count, public
    inputs as 32 B words or None, proofs as 256 B rows, or as 128 B rows when compressed)"""
    args = _batch_args(fn, vk, public_inputs, proofs, compressed)
    if args is None:
        return None
    ctx = ctx or default_context()
    return (ctx, ctx.vk_handle(vk)) + args


def _batch_args(fn, vk, public_inputs, proofs, compressed):
    """_verify_args without the device key: None for an empty batch, else (count, public inputs, proof rows)"""
    from . import verifier
    public_inputs, proofs = [list(x) for x in public_inputs], list(proofs)
    if len(public_inputs) != len(proofs):
        raise ValueError(f"{fn}: one public-input list per proof")
    if not proofs:
        return None
    rows = _proof_rows(fn, proofs, compressed)
    base = vk.vk if isinstance(vk, verifier.PreparedVerifyingKey) else vk
    n_public = len(base.gamma_abc_g1) - 1
    for xs in public_inputs:
        if len(xs) != n_public:
            raise verifier.MalformedVerifyingKey(f"{len(xs)} public inputs for a key with {n_public}")
        for x in xs:
            if not 0 <= int(x) < R_MOD:        # the library refuses >= r too; this also covers values no 32 B word holds
                raise N.B2gError(N.B2G_E_INPUT, f"public input {int(x)} is not in [0, r)")
    pub = b''.join(int(x).to_bytes(32, 'little') for xs in public_inputs for x in xs)
    pub_arr = np.frombuffer(pub, dtype=np.uint8).copy() if pub else None
    data = np.frombuffer(rows, dtype=np.uint8).copy()
    return len(proofs), pub_arr, data


# the library entry of each verifier, by (kind, compressed)
_VERIFY_ENTRY = {(kind, compressed): f"b2g_verify_{kind}{'_compressed' if compressed else ''}"
                 for kind in ('many', 'batch', 'batch_locate', 'batch_keys', 'batch_keys_locate') for compressed in (False, True)}


def _check_weights(where, weights, count, at=''):
    """caller-given weights as ints, one per proof and each in [1, 2^128), checked before the key is loaded on the device;
    `at` starts the message of a weight out of range"""
    weights = [int(w) for w in weights]
    if len(weights) != count:
        raise ValueError(f"{where}: one weight per proof")
    for w in weights:
        if not 0 < w < 1 << 128:
            raise N.B2gError(N.B2G_E_INPUT, f"{at}weight {w} is not in [1, 2^128)")
    return weights


def _weight_bytes(weights, count) -> np.ndarray:
    """the weights as 16-byte little-endian words, drawn with secrets.randbits(128) (never 0) when None"""
    import secrets
    if weights is None:
        weights = []
        while len(weights) < count:
            w = secrets.randbits(128)
            if w:
                weights.append(w)
    return np.frombuffer(b''.join(w.to_bytes(16, 'little') for w in weights), dtype=np.uint8).copy()


def _verify_one_key(fn, kind, vk, public_inputs, proofs, ctx, compressed, weights=None):
    """Groth16.verify_many, verify_batch, verify_batch_locate and their compressed forms (kind 'many', 'batch' or
    'batch_locate'): one bool for 'batch', else one bool per proof"""
    proofs = list(proofs)
    if weights is not None:
        weights = _check_weights(fn, weights, len(proofs))
    args = _verify_args(fn, vk, public_inputs, proofs, ctx, compressed)
    if args is None:
        return True if kind == 'batch' else []
    ctx, vh, count, pub_arr, data = args
    wb = None if kind == 'many' else _weight_bytes(weights, count)
    out = np.zeros(1 if kind == 'batch' else count, dtype=np.uint8)
    ws = () if wb is None else (_ptr(wb),)
    N.check(getattr(N.lib(), _VERIFY_ENTRY[kind, compressed])(ctx._h, vh, count, _ptr(pub_arr), _ptr(data), *ws, _ptr(out)))
    return bool(out[0]) if kind == 'batch' else [bool(v) for v in out]


def _key_batches(fn, batches, ctx, weights, compressed):
    """the argument checks and encoding of the keyed verifiers: (ctx, number of batches, [(batch index, KeyBatch)] for the
    batches that hold proofs, the arrays the KeyBatch rows point into).
    Every batch's checks run first, in batch order, up to the first batch j that fails them (j = the number of batches when
    none fails).  The keys of the batches before j that hold proofs and are not yet on the device then load in ONE
    b2g_vk_load_many call.  A key the library refuses raises under the lowest batch that uses it; otherwise batch j raises
    its own error.  So the errors, and which of them wins, are those of loading each batch's key as the batch is reached."""
    from . import verifier
    batches = [tuple(b) for b in batches]
    for k, b in enumerate(batches):
        if len(b) != 3:
            raise ValueError(f"{fn}: key {k}: a batch is (vk, public_inputs, proofs)")
    if weights is not None:
        weights = [None if w is None else [int(x) for x in w] for w in weights]
        if len(weights) != len(batches):
            raise ValueError(f"{fn}: one weight list per key batch")
    ctx = ctx or default_context()
    checked, loads, first_use, failure = [], {}, {}, None
    for k, (vk, public_inputs, proofs) in enumerate(batches):
        where = f"{fn}: key {k}"
        try:
            proofs = list(proofs)
            ws = None if weights is None else weights[k]
            if ws is not None:
                _check_weights(where, ws, len(proofs), f"{where}: ")
            try:
                args = _batch_args(where, vk, public_inputs, proofs, compressed)
                cache_key = (id(vk), ctx.device)
                if args is not None and cache_key not in _VK_HANDLES and cache_key not in loads:
                    loads[cache_key] = (vk,) + _vk_desc(vk)
                    first_use[cache_key] = k
            except N.B2gError as e:
                raise N.B2gError(e.code, f"{where}: {e.msg}") from e
            except verifier.MalformedVerifyingKey as e:
                raise verifier.MalformedVerifyingKey(f"{where}: {e}") from e
        except Exception as e:                 # raised once the keys of the batches before this one are loaded
            failure = e
            break
        if args is not None:                   # an empty batch is not passed on
            checked.append((k, vk, ws, args))
    try:
        ctx._vk_load_many(list(loads.values()))
    except N.B2gError as e:
        i, msg = _refused_key(e)
        k = first_use[list(loads)[i or 0]]
        raise N.B2gError(e.code, f"{fn}: key {k}: {msg}") from e
    if failure is not None:
        raise failure
    rows, keep = [], []
    for k, vk, ws, (count, pub_arr, data) in checked:
        vh = _VK_HANDLES[(id(vk), ctx.device)][0]
        wb = _weight_bytes(ws, count)
        keep += [pub_arr, data, wb]
        rows.append((k, N.KeyBatch(vh.value, count, 0, _ptr(pub_arr).value if pub_arr is not None else None, _ptr(data).value,
                                   _ptr(wb).value)))
    return ctx, len(batches), rows, keep


def _verify_batch_keys(fn, batches, ctx, weights, compressed, locate) -> list:
    """Groth16.verify_batch_keys, verify_batch_keys_locate and their compressed forms: per (vk, public_inputs, proofs)
    batch one bool, or one list of bools when locate"""
    ctx, n, rows, keep = _key_batches(fn, batches, ctx, weights, compressed)
    verdicts = [[] if locate else True for _ in range(n)]      # an empty batch has no verdicts, or is True
    if not rows:
        return verdicts
    table = (N.KeyBatch * len(rows))(*[r for _, r in rows])
    out = np.zeros(sum(r.count for _, r in rows) if locate else len(rows), dtype=np.uint8)
    entry = getattr(N.lib(), _VERIFY_ENTRY['batch_keys_locate' if locate else 'batch_keys', compressed])
    N.check(entry(ctx._h, len(rows), table, _ptr(out)))
    at = 0
    for i, (k, r) in enumerate(rows):
        verdicts[k] = [bool(v) for v in out[at:at + r.count]] if locate else bool(out[i])
        at += r.count
    return verdicts


def _scalar_bytes(v) -> np.ndarray:
    if isinstance(v, (int, np.integer)):
        return np.frombuffer((int(v) % R_MOD).to_bytes(32, 'little'), dtype='<u8').copy()
    a = _c(v).reshape(-1)
    if a.size != 4:
        raise ValueError("scalar must be an int or 4 uint64 limbs (canonical)")
    return a


def _prove_inputs(n_vars: int, rs, assignments, what: str = ''):
    """the witnesses of a prove call as contiguous arrays and its (r, s) as canonical limbs, r and s of every proof side by
    side; a witness of another length than n_vars raises ValueError (prefixed with `what`)"""
    ws = [_c(w) for w in assignments]
    for w in ws:
        if w.size // 4 != n_vars:
            raise ValueError(what + "full_assignment length != n_vars")
    return ws, [_scalar_bytes(r) for r, _ in rs], [_scalar_bytes(s) for _, s in rs]


def fr_rand(rng) -> int:
    """Fr::rand of ark-ff 0.5 (SURVEY.md App. C.5), the rule Groth16::prove uses for r and s: four u64 limbs from the rng
    (limb 0 first), the top two bits of limb 3 cleared, rejected and redrawn if >= r, and the limbs taken AS the Montgomery
    representation (value = limbs * R^-1 mod r).  `rng` supplies 64-bit words through next_u64() if it has one (an adapter
    over a rand-compatible stream), else through getrandbits(64) (random.Random, secrets.SystemRandom).  Same rule as
    ark_circom::Fr::rand in the C++ mirror."""
    nxt = rng.next_u64 if hasattr(rng, 'next_u64') else (lambda: rng.getrandbits(64))
    while True:
        limbs = [nxt() & 0xFFFFFFFFFFFFFFFF for _ in range(4)]
        limbs[3] &= 0x3FFFFFFFFFFFFFFF
        v = sum(x << (64 * i) for i, x in enumerate(limbs))
        if v < R_MOD:
            return v * _R_INV_R % R_MOD


_R_INV_R = pow(1 << 256, -1, R_MOD)


def _rerandomize_factors(rng) -> tuple:
    """(r1, r2) as Groth16::rerandomize_proof (ark-groth16 0.5.0) draws them: r1 = Fr::rand, then r2 = Fr::rand (fr_rand),
    both drawn again while either is zero"""
    r1 = r2 = 0
    while r1 == 0 or r2 == 0:
        r1 = fr_rand(rng)
        r2 = fr_rand(rng)
    return r1, r2


def _mont_points(points, g2: bool) -> np.ndarray:
    """canonical affine points (None = infinity) -> rows of Montgomery words, all-zero = infinity"""
    from .zkey import Q_MOD
    vals = []
    for pt in points:
        coords = ([0] * (4 if g2 else 2) if pt is None else
                  [pt[0][0], pt[0][1], pt[1][0], pt[1][1]] if g2 else [pt[0], pt[1]])
        vals += [0 if pt is None else (int(v) << 256) % Q_MOD for v in coords]
    return np.frombuffer(b''.join(v.to_bytes(32, 'little') for v in vals), dtype='<u8').copy()


def _circuit_desc(circuit, reduction):
    """(b2g_mat_desc with C, the arrays it points into, n_vars, num_inputs, the domain size, the H query's size) of a
    synth.Circuit or ConstraintMatrices with C, as the setup takes them"""
    m, n_vars = (circuit.matrices(with_c=True), circuit.n_vars) if hasattr(circuit, 'matrices') else (circuit, circuit.n_vars)
    d, keep = _mat_desc(m, n_vars, reduction.ID, with_c=True)
    ni = m.num_instance_variables
    if ni == 0 or ni > n_vars:
        raise N.B2gError(N.B2G_E_SHAPE, "num_inputs out of range")
    size = 1
    while size < m.num_constraints + ni:
        size <<= 1
    return d, keep, n_vars, ni, size, size - 1 if reduction.ID == N.REDUCTION_LIBSNARK else size


def _powers_desc(powers, size):
    """(b2g_powers_desc, the arrays it points into) of the prefix of a ceremony a domain of `size` points reads, as views where
    they can be; ValueError when an array is shorter.  A domain above the ceremony's power is left for the library to refuse
    before it reads any point."""
    from .ptau import ARRAYS, Powers
    log_n = size.bit_length() - 1
    pd = N.PowersDesc()
    pd.log_size = int(powers.power)
    arrays = {}
    if log_n <= pd.log_size:
        pre = Powers(int(powers.power), int(getattr(powers, 'ceremony_power', powers.power)),
                     *(np.asarray(getattr(powers, k)) for k in ARRAYS)).prefix(log_n)
        for name in ARRAYS:
            a = _c(getattr(pre, name))
            arrays[name] = a
            setattr(pd, name, a.ctypes.data)
    return pd, arrays


def _lagrange_descs(powers, log_n):
    """(b2g_powers_desc, b2g_lagrange_desc, the arrays they point into) of the prefix a domain of 2^log_n points reads from a
    ceremony with prepared Lagrange sections (tau_g1 with 2n points below the prepared power: the top block reads them)"""
    from .ptau import ARRAYS, LAGRANGE, Powers
    pre = Powers(int(powers.power), int(getattr(powers, 'ceremony_power', powers.power)),
                 *(np.asarray(getattr(powers, k)) for k in ARRAYS), lagrange=powers.lagrange).prefix(log_n)
    pd, ld, keep = N.PowersDesc(), N.LagrangeDesc(), []
    pd.log_size, ld.log_size = int(powers.power), int(pre.lagrange.power)
    for desc, src, names in ((pd, pre, ARRAYS), (ld, pre.lagrange, LAGRANGE)):
        for name in names:
            a = _c(getattr(src, name))
            keep.append(a)
            setattr(desc, name, a.ctypes.data)
    return pd, ld, keep


def _delta_desc(arrs) -> 'N.DeltaKey':
    d = N.DeltaKey()
    d.n_l, d.n_h = arrs['l_query'].size // 8, arrs['h_query'].size // 8
    for name, a in arrs.items():
        setattr(d, name, a.ctypes.data if a.size else None)
    return d


def _delta_key(pk: ProvingKey):
    """(b2g_delta_key of the key's delta, L and H fields, the arrays it points into)"""
    keep = {name: _c(getattr(pk, name)).reshape(-1, 16 if name == 'delta_g2' else 8)
            for name in ('delta_g1', 'delta_g2', 'l_query', 'h_query')}
    return _delta_desc(keep), keep


class CircomReduction:
    """R1CSToQAP implementation selected by Groth16<Bn254, CircomReduction> (src/circom/qap.rs:12-14)."""
    ID = N.REDUCTION_CIRCOM

    @classmethod
    def witness_map_from_matrices(cls, matrices: ConstraintMatrices, num_inputs: int, num_constraints: int, full_assignment, ctx: Context = None) -> np.ndarray:
        ctx = ctx or default_context()
        if num_inputs != matrices.num_instance_variables or num_constraints != matrices.num_constraints:
            raise ValueError("num_inputs / num_constraints disagree with the matrices")
        w = _c(full_assignment)
        n_vars = w.size // 4
        mh = ctx.mat_handle(matrices, n_vars, cls.ID)
        n = 1
        while n < num_constraints + num_inputs:
            n <<= 1
        h = np.zeros((n, 4), dtype=np.uint64)
        dom = C.c_uint32()
        N.check(N.lib().b2g_witness_map(ctx._h, mh, _ptr(w), _ptr(h), C.byref(dom)))
        assert dom.value == n
        return h


class LibsnarkReduction(CircomReduction):
    """ark-groth16's default R1CSToQAP (`Groth16<Bn254>` in /root/reference/tests/groth16.rs:9,25-35): h = coefficients of
    (a*b - c)/Z, c from the real C matrix; keys from generate_random_parameters_with_reduction carry domain_size - 1 H bases."""
    ID = N.REDUCTION_LIBSNARK


class Groth16:
    """Groth16::<Bn254, QAP>; QAP = CircomReduction (snarkjs keys, default here) or LibsnarkReduction (arkworks keys)."""

    @staticmethod
    def create_proof_with_reduction_and_matrices(pk: ProvingKey, r, s, matrices: ConstraintMatrices, num_inputs: int,
                                                 num_constraints: int, full_assignment, ctx: Context = None, reduction=CircomReduction) -> Proof:
        ctx = ctx or default_context()
        if num_inputs != matrices.num_instance_variables or num_constraints != matrices.num_constraints:
            raise ValueError("num_inputs / num_constraints disagree with the matrices")
        (w,), (rr,), (ss,) = _prove_inputs(pk.n_vars, [(r, s)], [full_assignment])
        ph, mh = ctx.pk_handle(pk), ctx.mat_handle(matrices, pk.n_vars, reduction.ID)
        out = np.zeros(256, dtype=np.uint8)
        N.check(N.lib().b2g_prove(ctx._h, ph, mh, _ptr(rr), _ptr(ss), _ptr(w), _ptr(out)))
        return Proof(out.tobytes())

    @staticmethod
    def create_proofs(pk: ProvingKey, rs, matrices: ConstraintMatrices, assignments, ctx: Context = None, reduction=CircomReduction) -> list:
        """create_proof_with_reduction_and_matrices for many witnesses of one circuit in ONE device pass (b2g_prove_many):
        rs = sequence of (r, s), assignments = sequence of Montgomery full assignments; returns [Proof], proof i byte-identical
        to the single call with (r_i, s_i, assignments[i]).  Unlike K contexts with submit / wait, every kernel of the
        pipeline runs once for the whole batch; the context keeps device buffers for the largest batch it has proved."""
        ctx = ctx or default_context()
        rs, assignments = list(rs), list(assignments)
        if len(rs) != len(assignments):
            raise ValueError("create_proofs: one (r, s) per assignment")
        if not assignments:
            return []
        ws, rr, ss = _prove_inputs(pk.n_vars, rs, assignments)
        ph, mh = ctx.pk_handle(pk), ctx.mat_handle(matrices, pk.n_vars, reduction.ID)
        rr, ss = np.concatenate(rr), np.concatenate(ss)
        ptrs = (C.c_void_p * len(ws))(*[w.ctypes.data for w in ws])
        out = np.zeros((len(ws), 256), dtype=np.uint8)
        N.check(N.lib().b2g_prove_many(ctx._h, ph, mh, len(ws), _ptr(rr), _ptr(ss), ptrs, _ptr(out)))
        return [Proof(row.tobytes()) for row in out]

    @staticmethod
    def load_proving_keys(keys, ctx: Context = None, reduction=CircomReduction) -> ProvingKeyGroup:
        """Loads keys = [(pk, matrices) or (pk, matrices, reduction), ...] on ctx's device for create_proofs_keys
        (b2g_pk_group_load): every query's tables of all keys in one arena at one window size.  A key may appear more than
        once; `reduction` applies to the pairs that name none.  Returns the group, freed by release(group).  A key the
        library refuses raises B2gError naming its index; then nothing is loaded."""
        ctx = ctx or default_context()
        entries = [tuple(e) if len(e) == 3 else (e[0], e[1], reduction) for e in keys]
        if not entries:
            raise ValueError("load_proving_keys: the group has no keys")
        descs, keep, mats, owned = [], [], [], {}
        try:
            for pk, m, red in entries:
                d, k = _pk_desc(pk)
                descs.append(d)
                keep.append(k)
                if (id(m), red.ID) not in owned:
                    md, mk = _mat_desc(m, pk.n_vars, red.ID)
                    h = C.c_void_p()
                    N.check(N.lib().b2g_matrices_load(ctx._h, C.byref(md), C.byref(h)))
                    owned[(id(m), red.ID)] = h
                mats.append(owned[(id(m), red.ID)])
            arr = (N.PkDesc * len(descs))(*descs)
            hs = (C.c_void_p * len(mats))(*[h.value for h in mats])
            g = C.c_void_p()
            N.check(N.lib().b2g_pk_group_load(ctx._h, len(descs), arr, hs, C.byref(g)))
        except BaseException:
            for h in owned.values():
                N.lib().b2g_matrices_free(h)
            raise
        return ProvingKeyGroup(ctx.device, [(pk, m, red) for pk, m, red in entries], g, list(owned.values()))

    @staticmethod
    def create_proofs_keys(group: ProvingKeyGroup, batches, ctx: Context = None) -> list:
        """create_proofs for one batch per key of `group`, all in ONE device pass (b2g_prove_keys): batches = one
        (rs, assignments) per key, in the group's order (an empty batch is allowed); returns one [Proof] per key, batch k's
        proofs byte-identical to create_proofs(pk_k, rs_k, matrices_k, assignments_k)."""
        ctx = ctx or default_context()
        batches = [(list(rs), list(ws)) for rs, ws in batches]
        if len(batches) != group.n_keys:
            raise ValueError(f"create_proofs_keys: {len(batches)} batches for a group of {group.n_keys} keys")
        if not group._h:
            raise ValueError("create_proofs_keys: the group has been released")
        ws, rr, ss, counts = [], [], [], []
        for k, ((rs, assignments), (pk, _, _)) in enumerate(zip(batches, group.keys)):
            if len(rs) != len(assignments):
                raise ValueError(f"create_proofs_keys: key {k}: one (r, s) per assignment")
            kw, kr, ks = _prove_inputs(pk.n_vars, rs, assignments, f"create_proofs_keys: key {k}: ")
            ws += kw
            rr += kr
            ss += ks
            counts.append(len(assignments))
        if not ws:
            return [[] for _ in batches]
        cnt = np.array(counts, dtype=np.uint32)
        rr, ss = np.concatenate(rr), np.concatenate(ss)
        ptrs = (C.c_void_p * len(ws))(*[w.ctypes.data for w in ws])
        out = np.zeros((len(ws), 256), dtype=np.uint8)
        N.check(N.lib().b2g_prove_keys(ctx._h, group._h, _ptr(cnt), _ptr(rr), _ptr(ss), ptrs, _ptr(out)))
        proofs, at = [], 0
        for c in counts:
            proofs.append([Proof(row.tobytes()) for row in out[at:at + c]])
            at += c
        return proofs

    @staticmethod
    def submit(pk: ProvingKey, r, s, matrices: ConstraintMatrices, full_assignment, ctx: Context, reduction=CircomReduction) -> 'PendingProof':
        """create_proof_with_reduction_and_matrices without the wait: enqueues the proof on `ctx` (one pending proof per
        context) and returns a handle whose .wait() yields the Proof.  One host thread + K contexts = K proofs in flight."""
        (w,), (rr,), (ss,) = _prove_inputs(pk.n_vars, [(r, s)], [full_assignment])
        ph, mh = ctx.pk_handle(pk), ctx.mat_handle(matrices, pk.n_vars, reduction.ID)
        out = np.zeros(256, dtype=np.uint8)
        N.check(N.lib().b2g_prove_submit(ctx._h, ph, mh, _ptr(rr), _ptr(ss), _ptr(w), _ptr(out)))
        return PendingProof(ctx, out, w)

    @staticmethod
    def prove(pk: ProvingKey, matrices: ConstraintMatrices, full_assignment, rng, ctx: Context = None, reduction=CircomReduction) -> Proof:
        """Draws r then s like create_random_proof_with_reduction (ark-groth16 0.5.0), each with the Fr::rand limb rule
        (fr_rand above): fed the same u64 stream as a seeded arkworks rng, it proves with the same (r, s)."""
        r = fr_rand(rng)
        s = fr_rand(rng)
        return Groth16.create_proof_with_reduction_and_matrices(pk, r, s, matrices, matrices.num_instance_variables,
                                                                matrices.num_constraints, full_assignment, ctx, reduction)

    @staticmethod
    def generate_random_parameters_with_reduction(circuit, rng, ctx: Context = None, reduction=CircomReduction) -> ProvingKey:
        """Setup on the GPU (tests/groth16.rs:25 flow): the toxic waste alpha, beta, gamma, delta, tau is drawn in that order
        with rng.randrange(1, r), the key is built on the standard generators by one b2g_setup call, and the toxic waste is
        dropped.  `circuit` is a synth.Circuit (R1CS as coordinate lists) or ConstraintMatrices with C."""
        alpha, beta, gamma, delta, tau = (rng.randrange(1, R_MOD) for _ in range(5))
        return Groth16.generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, tau=tau, ctx=ctx, reduction=reduction)

    @staticmethod
    def generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, g1_generator=None, g2_generator=None, *, tau,
                                     ctx: Context = None, reduction=CircomReduction) -> ProvingKey:
        """Groth16::generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, g1_generator, g2_generator, rng)
        (ark-groth16 0.5) with tau given instead of drawn from the rng; every scalar and point is computed on the GPU by
        b2g_setup.  Scalars are ints in [0, r) (gamma, delta nonzero); generators are in the ProvingKey point-array layout
        (8 / 16 uint64 words, affine Montgomery), None for the standard ones.  `circuit` is a synth.Circuit or
        ConstraintMatrices with C (the R1CS route); its n_vars is then the matrices' own."""
        ctx = ctx or default_context()
        if hasattr(circuit, 'matrices'):
            m, n_vars = circuit.matrices(with_c=True), circuit.n_vars
        else:
            m, n_vars = circuit, circuit.n_vars
        d, keep = _mat_desc(m, n_vars, reduction.ID, with_c=True)
        ni = m.num_instance_variables
        if ni == 0 or ni > n_vars:
            raise N.B2gError(N.B2G_E_SHAPE, "num_inputs out of range")
        size = 1
        while size < m.num_constraints + ni:
            size <<= 1
        nh = size - 1 if reduction.ID == N.REDUCTION_LIBSNARK else size
        secrets = np.frombuffer(b''.join(int(v).to_bytes(32, 'little') for v in (alpha, beta, gamma, delta, tau)), dtype=np.uint8).copy()
        sec = N.SetupSecrets()
        for i, name in enumerate(('alpha', 'beta', 'gamma', 'delta', 'tau')):
            setattr(sec, name, secrets.ctypes.data + 32 * i)
        gens = []
        for name, gen, words in (('g1', g1_generator, 8), ('g2', g2_generator, 16)):
            if gen is not None:
                g = _c(gen).reshape(-1)
                if g.size != words:
                    raise ValueError(f"{name}_generator must be {words} uint64 words (affine Montgomery)")
                gens.append(g)
                setattr(sec, name, g.ctypes.data)
        shapes = {'alpha_g1': (1, 8), 'beta_g1': (1, 8), 'delta_g1': (1, 8), 'beta_g2': (1, 16), 'gamma_g2': (1, 16), 'delta_g2': (1, 16),
                  'gamma_abc_g1': (ni, 8), 'a_query': (n_vars, 8), 'b_g1_query': (n_vars, 8), 'b_g2_query': (n_vars, 16),
                  'l_query': (n_vars - ni, 8), 'h_query': (nh, 8)}
        arrs = {k: np.zeros(v, dtype=np.uint64) for k, v in shapes.items()}
        out = N.SetupOut()
        for k, a in arrs.items():
            setattr(out, k, a.ctypes.data if a.size else None)
        try:
            N.check(N.lib().b2g_setup(ctx._h, C.byref(d), C.byref(sec), C.byref(out)))
        finally:
            secrets[:] = 0
        return ProvingKey(n_vars, ni - 1, nh, arrs['alpha_g1'], arrs['beta_g1'], arrs['beta_g2'], arrs['gamma_g2'], arrs['delta_g1'],
                          arrs['delta_g2'], arrs['gamma_abc_g1'], arrs['a_query'], arrs['b_g1_query'], arrs['b_g2_query'],
                          arrs['l_query'], arrs['h_query'])

    @staticmethod
    def generate_parameters_from_powers_of_tau(circuit, powers, ctx: Context = None, reduction=CircomReduction) -> ProvingKey:
        """`snarkjs groth16 setup circuit.r1cs pot.ptau` on the GPU (b2g_setup_from_powers): the proving key of `circuit` (as
        generate_parameters_with_qap takes it) from a powers-of-tau ceremony (ptau.read_ptau, or any object with the same
        fields), with gamma = delta = 1.  Only the prefix of each array the circuit's domain needs is read.  A ceremony that
        carries prepared Lagrange sections (powers.lagrange, as read_ptau attaches them) takes b2g_setup_from_lagrange, which
        reads the Lagrange points instead of transforming the powers and gives the same key when the sections are honest
        (verify_powers_of_tau checks them); any other takes b2g_setup_from_powers."""
        ctx = ctx or default_context()
        d, keep, n_vars, ni, size, nh = _circuit_desc(circuit, reduction)
        lag = getattr(powers, 'lagrange', None)
        if lag is not None and size.bit_length() - 1 <= min(int(powers.power), int(lag.power)):
            pd, ld, arrays = _lagrange_descs(powers, size.bit_length() - 1)
        else:
            ld = None
            pd, arrays = _powers_desc(powers, size)
        shapes = {'alpha_g1': (1, 8), 'beta_g1': (1, 8), 'delta_g1': (1, 8), 'beta_g2': (1, 16), 'gamma_g2': (1, 16), 'delta_g2': (1, 16),
                  'gamma_abc_g1': (ni, 8), 'a_query': (n_vars, 8), 'b_g1_query': (n_vars, 8), 'b_g2_query': (n_vars, 16),
                  'l_query': (n_vars - ni, 8), 'h_query': (nh, 8)}
        arrs = {k: np.zeros(v, dtype=np.uint64) for k, v in shapes.items()}
        out = N.SetupOut()
        for k, a in arrs.items():
            setattr(out, k, a.ctypes.data if a.size else None)
        if ld is not None:
            N.check(N.lib().b2g_setup_from_lagrange(ctx._h, C.byref(d), C.byref(pd), C.byref(ld), C.byref(out)))
        else:
            N.check(N.lib().b2g_setup_from_powers(ctx._h, C.byref(d), C.byref(pd), C.byref(out)))
        return ProvingKey(n_vars, ni - 1, nh, arrs['alpha_g1'], arrs['beta_g1'], arrs['beta_g2'], arrs['gamma_g2'], arrs['delta_g1'],
                          arrs['delta_g2'], arrs['gamma_abc_g1'], arrs['a_query'], arrs['b_g1_query'], arrs['b_g2_query'],
                          arrs['l_query'], arrs['h_query'])

    @staticmethod
    def verify_proving_key(circuit, powers, pk: ProvingKey, matrices: ConstraintMatrices = None, reduction=CircomReduction,
                           ctx: Context = None, challenges=None):
        """`snarkjs zkey verify circuit.r1cs pot.ptau circuit.zkey` on the GPU (b2g_setup_check), without snarkjs's transcript:
        whether `pk` is the key generate_parameters_from_powers_of_tau makes from `circuit` and `powers`, followed by any chain
        of `contribute` calls.  `circuit` and `powers` are what that call takes; `matrices`, the ConstraintMatrices read_zkey
        returns with the key, must then hold the circuit's A and B (compared on the host, row by row in canonical form) and its
        counts.  The key and the ceremony are read from host memory once, memory-mapped views in place.  The challenges rho
        and sigma (in [1, r)) are drawn with `secrets` unless given.  Returns a keycheck.SetupCheck: truthy when the key
        passes, .reason naming the first failing check.  A key that is not the circuit's passes with probability at most
        max(n_vars, n) / (r - 1) when the challenges are drawn after the key and the ceremony are fixed."""
        import secrets
        from .keycheck import KEY_FIELDS, SetupCheck, matrices_reason, report_reason, shape_reason
        d, keep, n_vars, ni, size, nh = _circuit_desc(circuit, reduction)
        if matrices is not None:
            why = matrices_reason(circuit.matrices() if hasattr(circuit, 'matrices') else circuit, matrices)
            if why:
                return SetupCheck(False, why)
        arrs = {k: _c(getattr(pk, k)).reshape(-1, 16 if k in ('beta_g2', 'gamma_g2', 'delta_g2', 'b_g2_query') else 8)
                for k in KEY_FIELDS}
        want = {'alpha_g1': 1, 'beta_g1': 1, 'delta_g1': 1, 'beta_g2': 1, 'gamma_g2': 1, 'delta_g2': 1, 'gamma_abc_g1': ni,
                'a_query': n_vars, 'b_g1_query': n_vars, 'b_g2_query': n_vars, 'l_query': n_vars - ni, 'h_query': nh}
        for k in KEY_FIELDS:
            if arrs[k].shape[0] != want[k]:
                return SetupCheck(False, shape_reason(k, arrs[k].shape[0], want[k], reduction.__name__, size))
        pd, arrays = _powers_desc(powers, size)
        if challenges is None:
            challenges = [1 + secrets.randbelow(R_MOD - 1) for _ in range(2)]
        challenges = [int(c) for c in challenges]
        if len(challenges) != 2 or not all(0 <= c < 1 << 256 for c in challenges):
            raise ValueError("verify_proving_key: two challenges (rho, sigma), each below 2^256")
        cb = np.frombuffer(b''.join(c.to_bytes(32, 'little') for c in challenges), dtype=np.uint8).copy()
        kd = N.KeyDesc()
        kd.n_vars, kd.n_ic, kd.n_l, kd.n_h = n_vars, ni, n_vars - ni, nh
        for k, a in arrs.items():
            setattr(kd, k, a.ctypes.data if a.size else None)
        rep = N.SetupReport()
        ctx = ctx or default_context()
        N.check(N.lib().b2g_setup_check(ctx._h, C.byref(d), C.byref(pd), C.byref(kd), _ptr(cb), C.byref(rep)))
        return SetupCheck(True) if rep.ok else SetupCheck(False, report_reason(rep))

    @staticmethod
    def contribute(pk: ProvingKey, rng=None, ctx: Context = None, x=None) -> ProvingKey:
        """`snarkjs zkey contribute` on the GPU (b2g_delta_update): a new key with delta multiplied by a secret x and the L and
        H queries divided by it.  x is drawn in [1, r) with `secrets` (or rng.randrange when an rng is given) unless given;
        it is not returned, and the library's copies of it are wiped."""
        import secrets
        ctx = ctx or default_context()
        if x is None:
            x = rng.randrange(1, R_MOD) if rng is not None else 1 + secrets.randbelow(R_MOD - 1)
        x = int(x)
        if not 0 <= x < 1 << 256:
            raise N.B2gError(N.B2G_E_INPUT, "x is not below r")
        xb = np.frombuffer(x.to_bytes(32, 'little'), dtype=np.uint8).copy()
        before, keep = _delta_key(pk)
        after_arrs = {'delta_g1': np.zeros((1, 8), dtype=np.uint64), 'delta_g2': np.zeros((1, 16), dtype=np.uint64),
                      'l_query': np.zeros_like(keep['l_query']), 'h_query': np.zeros_like(keep['h_query'])}
        after = _delta_desc(after_arrs)
        try:
            N.check(N.lib().b2g_delta_update(ctx._h, C.byref(before), _ptr(xb), C.byref(after)))
        finally:
            xb[:] = 0
        return ProvingKey(pk.n_vars, pk.n_public, pk.domain_size, np.array(pk.alpha_g1, copy=True), np.array(pk.beta_g1, copy=True),
                          np.array(pk.beta_g2, copy=True), np.array(pk.gamma_g2, copy=True), after_arrs['delta_g1'], after_arrs['delta_g2'],
                          np.array(pk.gamma_abc_g1, copy=True), np.array(pk.a_query, copy=True), np.array(pk.b_g1_query, copy=True),
                          np.array(pk.b_g2_query, copy=True), after_arrs['l_query'], after_arrs['h_query'])

    @staticmethod
    def verify_contribution(before: ProvingKey, after: ProvingKey, ctx: Context = None, weights=None) -> bool:
        """The delta checks of `snarkjs zkey verify` (b2g_delta_update_check): whether `after` is `before` with one or more
        delta contributions.  The fields a contribution leaves alone are compared on the host; the weights (one per L point,
        then one per H point, in [1, 2^128)) are drawn with `secrets` unless given.  A False verdict is wrong with probability
        at most 1 / (2^128 - 1) per equation when the weights are drawn after both keys are fixed."""
        ctx = ctx or default_context()
        for name in ('n_vars', 'n_public', 'domain_size'):
            if getattr(before, name) != getattr(after, name):
                return False
        for name in ('alpha_g1', 'beta_g1', 'beta_g2', 'gamma_g2', 'gamma_abc_g1', 'a_query', 'b_g1_query', 'b_g2_query'):
            a, b = _c(getattr(before, name)), _c(getattr(after, name))
            if a.shape != b.shape or a.tobytes() != b.tobytes():
                return False
        d0, k0 = _delta_key(before)
        d1, k1 = _delta_key(after)
        if (d0.n_l, d0.n_h) != (d1.n_l, d1.n_h):
            return False
        count = d0.n_l + d0.n_h
        if weights is not None:
            weights = _check_weights("verify_contribution", weights, count)
        wb = _weight_bytes(weights, count)
        out = np.zeros(1, dtype=np.uint8)
        N.check(N.lib().b2g_delta_update_check(ctx._h, C.byref(d0), C.byref(d1), _ptr(wb), _ptr(out)))
        return bool(out[0])

    @staticmethod
    def prepare_powers_of_tau(powers, dst=None, power=None, ctx: Context = None):
        """`snarkjs powersoftau prepare phase2` on the GPU (b2g_powers_prepare): the ceremony of power K (`power`, by default
        min(powers.power, 26)) formed by the prefix of `powers`, with its Lagrange sections 12-15.  Returns a ptau.Powers with
        .lagrange set; with `dst` (a path) the prepared .ptau is written there, the sections filled in place through a memory
        map so that files larger than memory work, and the result is that file read back (memory-mapped).  The points read are
        checked as generate_parameters_from_powers_of_tau checks them; whether they are a ceremony is verify_powers_of_tau's
        question."""
        from .ptau import ARRAYS, LAGRANGE, Lagrange, Powers, lagrange_counts, read_ptau, write_ptau
        K = min(int(powers.power), 26) if power is None else int(power)
        if not 1 <= K <= min(int(powers.power), 26):
            raise ValueError(f"prepare_powers_of_tau: power {K} is outside 1..{min(int(powers.power), 26)}")
        pre = Powers(K, int(getattr(powers, 'ceremony_power', powers.power)),
                     *(np.asarray(getattr(powers, k)) for k in ARRAYS)).prefix(K)
        if dst is not None:
            write_ptau(dst, pre, lagrange_space=True)
            mm = np.memmap(dst, dtype=np.uint8, mode='r+')
            outs = [getattr(read_ptau(mm).lagrange, k) for k in LAGRANGE]
        else:
            mm = None
            outs = [np.zeros((c, 16 if k == 'tau_g2' else 8), dtype=np.uint64) for k, c in zip(LAGRANGE, lagrange_counts(K))]
        pd, keep = N.PowersDesc(), []
        pd.log_size = int(powers.power)
        for name in ARRAYS:
            a = _c(getattr(pre, name))
            keep.append(a)
            setattr(pd, name, a.ctypes.data)
        od = N.LagrangeDesc()
        od.log_size = K
        for name, a in zip(LAGRANGE, outs):
            setattr(od, name, a.ctypes.data)
        ctx = ctx or default_context()
        N.check(N.lib().b2g_powers_prepare(ctx._h, C.byref(pd), C.byref(od)))
        if mm is not None:
            mm.flush()
            del outs, mm
            return read_ptau(dst)
        return Powers(K, pre.ceremony_power, *(getattr(pre, k) for k in ARRAYS), lagrange=Lagrange(K, *outs))

    @staticmethod
    def contribute_powers_of_tau(powers, dst=None, rng=None, ctx: Context = None, tau=None, alpha=None, beta=None):
        """`snarkjs powersoftau contribute` on the GPU (b2g_powers_contribute): the ceremony of (tau t, alpha a, beta b) from
        the whole ceremony `powers` of (tau, alpha, beta), with the secrets t, a, b in [1, r) drawn with `secrets` (or
        rng.randrange when an rng is given) unless given.  The secrets are not returned and the byte buffers that carried them
        are wiped; the contribution is sound only if nobody keeps them.  Returns a ptau.Powers with the input's power and
        ceremony_power and no Lagrange sections (the input's no longer match).  With `dst` (a path) the container is written
        first and its sections filled in place through a memory map, so a ceremony larger than host memory streams, and the
        result is that file read back (memory-mapped).  Every point read is checked (on its curve, coordinates below p, not at
        infinity, tau_g1[0] and tau_g2[0] the generators, G2 points in G2); whether the input is a ceremony is
        verify_powers_of_tau's question, and verify_powers_of_tau on the output is the check of the result."""
        import secrets as _secrets
        from .ptau import ARRAYS, Powers, read_ptau, write_ptau
        power = int(powers.power)
        if not 1 <= power <= 28:
            raise ValueError(f"contribute_powers_of_tau: power {power} is outside 1..28")
        cp = int(getattr(powers, 'ceremony_power', power))
        pre = Powers(power, cp, *(np.asarray(getattr(powers, k)) for k in ARRAYS)).prefix(power)
        draw = (lambda: rng.randrange(1, R_MOD)) if rng is not None else (lambda: 1 + _secrets.randbelow(R_MOD - 1))
        vals = [draw() if v is None else int(v) for v in (tau, alpha, beta)]
        for name, v in zip(('tau', 'alpha', 'beta'), vals):
            if not 1 <= v < R_MOD:
                raise N.B2gError(N.B2G_E_INPUT, f"secret {name} is 0 or >= r")
        sb = np.frombuffer(b''.join(v.to_bytes(32, 'little') for v in vals), dtype=np.uint8).copy()
        del vals
        try:
            pd, keep = N.PowersDesc(), []
            pd.log_size = power
            for name in ARRAYS:
                a = _c(getattr(pre, name))
                keep.append(a)
                setattr(pd, name, a.ctypes.data)
            if dst is not None:
                write_ptau(dst, pre, points_space=True)
                mm = np.memmap(dst, dtype=np.uint8, mode='r+')
                res = read_ptau(mm)
                outs = [getattr(res, k) for k in ARRAYS]
            else:
                mm = None
                outs = [np.zeros_like(a) for a in keep]
            od = N.PowersOut()
            for name, a in zip(ARRAYS, outs):
                setattr(od, name, a.ctypes.data)
            sd = N.PowersSecrets()
            sd.tau, sd.alpha, sd.beta = sb.ctypes.data, sb.ctypes.data + 32, sb.ctypes.data + 64
            ctx = ctx or default_context()
            N.check(N.lib().b2g_powers_contribute(ctx._h, C.byref(pd), C.byref(sd), C.byref(od)))
        finally:
            sb[:] = 0
        if mm is not None:
            mm.flush()
            del outs, res, mm
            return read_ptau(dst)
        return Powers(power, cp, *outs)

    @staticmethod
    def verify_powers_of_tau(powers, log_n=None, ctx: Context = None, challenges=None):
        """The algebraic checks of `snarkjs powersoftau verify` on the GPU (b2g_powers_check): whether the prefix a domain of
        2^log_n points reads (the whole ceremony by default) holds powers of one tau with the same alpha and beta on the
        standard generators.  `powers` is a ptau.read_ptau result or any object with the same fields; memory-mapped views are
        read in place, once.  The five challenges (rho, sigma, pi, kappa, eps in [1, r)) are drawn with `secrets` unless
        given.  Returns a ptau.PowersCheck: truthy when the ceremony passes, .reason naming the first failing point or the
        failed pairing product.  A ceremony that is not one passes with probability at most 2n / (r - 1) when the challenges
        are drawn after the file is fixed.  Raises ValueError for a bad log_n or arrays shorter than it reads.
        When the ceremony carries prepared Lagrange sections (powers.lagrange) and passes, b2g_lagrange_check then decides
        whether their blocks up to log_n (log_n + 1 for lagrange_tau_g1) are the transforms of the powers, with one more
        challenge rho: the sixth entry of `challenges` when six are given, else drawn with `secrets`.  A wrong section passes
        with probability at most (its point count) / (r - 1); a failure's reason is "lagrange_tau_g2[17]: not in G2" or
        "lagrange_tau_g1 is not the transform of tau_g1"."""
        import secrets
        from .ptau import ARRAYS, REPORT_ARRAYS, Powers, PowersCheck
        power = int(powers.power)
        log_n = power if log_n is None else int(log_n)
        if log_n < 1:
            raise ValueError(f"verify_powers_of_tau: log_n {log_n} is below 1")
        pre = Powers(power, int(getattr(powers, 'ceremony_power', power)),
                     *(np.asarray(getattr(powers, k)) for k in ARRAYS)).prefix(log_n)
        if challenges is None:
            challenges = [1 + secrets.randbelow(R_MOD - 1) for _ in range(5)]
        challenges = [int(c) for c in challenges]
        if len(challenges) not in (5, 6) or not all(0 <= c < 1 << 256 for c in challenges):
            raise ValueError("verify_powers_of_tau: five challenges (rho, sigma, pi, kappa, eps), each below 2^256, and an "
                             "optional sixth for the Lagrange sections")
        cb = np.frombuffer(b''.join(c.to_bytes(32, 'little') for c in challenges[:5]), dtype=np.uint8).copy()
        pd = N.PowersDesc()
        pd.log_size = power
        keep = []
        for name in ARRAYS:
            a = _c(getattr(pre, name))
            keep.append(a)
            setattr(pd, name, a.ctypes.data)
        rep = N.PowersReport()
        ctx = ctx or default_context()
        N.check(N.lib().b2g_powers_check(ctx._h, C.byref(pd), log_n, _ptr(cb), C.byref(rep)))
        if rep.ok and getattr(powers, 'lagrange', None) is not None:
            rho = challenges[5] if len(challenges) == 6 else 1 + secrets.randbelow(R_MOD - 1)
            rb = np.frombuffer(int(rho).to_bytes(32, 'little'), dtype=np.uint8).copy()
            lpd, ld, keep = _lagrange_descs(powers, log_n)
            N.check(N.lib().b2g_lagrange_check(ctx._h, C.byref(lpd), C.byref(ld), log_n, _ptr(rb), C.byref(rep)))
        if rep.ok:
            return PowersCheck(True)
        if rep.rule == 6:
            return PowersCheck(False, 6)
        if rep.rule == 7:
            return PowersCheck(False, 7, REPORT_ARRAYS[rep.array])
        return PowersCheck(False, int(rep.rule), REPORT_ARRAYS[rep.array], int(rep.index))

    # ---- verification (host pairing; circom_compat_b200/verifier.py).  Call sites in the reference: src/zkey.rs:868-870,
    # 914-916 (process_vk + verify_with_processed_vk), tests/groth16.rs:33-35 (SNARK::verify).
    @staticmethod
    def process_vk(vk):
        """Groth16::process_vk(&params.vk): `vk` is a verifier.VerifyingKey or a ProvingKey (its vk part is used)."""
        from . import verifier
        return verifier.prepare_verifying_key(vk)

    @staticmethod
    def verify_with_processed_vk(pvk, public_inputs, proof) -> bool:
        """public_inputs = w[1..num_inputs] as integers (CircomCircuit::get_public_inputs, src/circom/circuit.rs:18-26)"""
        from . import verifier
        return verifier.verify_with_processed_vk(pvk, public_inputs, proof)

    @staticmethod
    def verify(vk, public_inputs, proof) -> bool:
        from . import verifier
        return verifier.verify(vk, public_inputs, proof)

    @staticmethod
    def verify_many(vk, public_inputs, proofs, ctx: Context = None) -> list:
        """verify_with_processed_vk for many proofs of one key in ONE device pass (b2g_verify_many): `vk` is a VerifyingKey,
        PreparedVerifyingKey or ProvingKey (prepared on the device once and cached per object), public_inputs = one
        sequence of ints per proof, proofs = [Proof].  Returns [bool].  Verdicts equal the host call's, except that a proof
        coordinate >= p is invalid here (arkworks cannot deserialise it) where the host verifier reduces it.  A public input
        outside [0, r) raises B2gError (B2G_E_INPUT); an input count that does not match the key raises MalformedVerifyingKey."""
        return _verify_one_key('verify_many', 'many', vk, public_inputs, proofs, ctx, False)

    @staticmethod
    def verify_batch(vk, public_inputs, proofs, ctx: Context = None, weights=None) -> bool:
        """Whether ALL proofs are valid, from one random-linear-combination pairing check on the device (b2g_verify_batch):
        cheaper per proof than verify_many, but one verdict for the batch.  On False, call verify_batch_locate to find the
        invalid proofs.  True iff every proof would pass verify_many, every B lies in G2 (verify_many does not check that), except
        with probability at most 1 / (2^128 - 1) when the weights are uniform.  Arguments and errors as verify_many; an empty
        batch is True.  `weights` (one int in [1, 2^128) per proof) are drawn with secrets.randbits(128) when not given;
        weights a prover could know or choose before fixing its proofs make the check unsound.  A zero or too large weight
        raises B2gError (B2G_E_INPUT)."""
        return _verify_one_key('verify_batch', 'batch', vk, public_inputs, proofs, ctx, False, weights)

    @staticmethod
    def verify_batch_locate(vk, public_inputs, proofs, ctx: Context = None, weights=None) -> list:
        """One verdict per proof at about verify_batch's cost when few proofs are invalid (b2g_verify_batch_locate).  The
        batch check runs once per group of 64 consecutive proofs, over the group's well-formed proofs (every coordinate
        below p, every point on its curve, B at infinity or in G2); the well-formed proofs of a group that fails it are
        then checked one by one as verify_many checks them.  A proof that is not well-formed is False.  A proof that
        verify_many accepts and whose B is in G2 is always True; any other proof is False except with probability at most
        (groups holding such a proof) / (2^128 - 1) when the weights are uniform.  Arguments, weights and errors as
        verify_batch; an empty batch gives []."""
        return _verify_one_key('verify_batch_locate', 'batch_locate', vk, public_inputs, proofs, ctx, False, weights)

    @staticmethod
    def load_verifying_keys(vks, ctx: Context = None) -> None:
        """Prepare many verifying keys on the device in ONE device pass (b2g_vk_load_many), e.g. when a node starts: every key
        (a VerifyingKey, PreparedVerifyingKey or ProvingKey) not yet on ctx's device is loaded and cached per object, as the
        verifiers cache it, so that no verifier call has to load it.  A key with a point off its curve raises B2gError
        (B2G_E_INPUT) naming its index in `vks`; then none of the keys is loaded.  release(vk) frees a key."""
        (ctx or default_context()).vk_handles(vks)

    @staticmethod
    def verify_batch_keys(batches, ctx: Context = None, weights=None) -> list:
        """verify_batch for many keys in ONE device pass (b2g_verify_batch_keys): batches = a sequence of (vk, public_inputs,
        proofs), each as verify_batch takes them (keys are prepared on the device once and cached per object, and one key
        may appear in several batches).  Returns one bool per batch, equal to verify_batch on that batch with the same
        weights; an invalid proof changes its own batch's verdict only, and an empty batch is True.  `weights` is None
        (drawn with secrets.randbits(128)) or one list per batch (None in it: drawn).  Argument checks and errors as
        verify_batch, with the batch's index in the message."""
        return _verify_batch_keys('verify_batch_keys', batches, ctx, weights, False, False)

    @staticmethod
    def verify_batch_keys_compressed(batches, ctx: Context = None, weights=None) -> list:
        """verify_batch_keys on compressed proofs (b2g_verify_batch_keys_compressed), decoded on the device: a batch with a
        blob that does not decode is False, and the other verdicts are those of verify_batch_keys on the decoded proofs.
        Arguments, weights and errors as verify_batch_keys; a blob that is not 128 bytes raises ValueError."""
        return _verify_batch_keys('verify_batch_keys_compressed', batches, ctx, weights, True, False)

    @staticmethod
    def verify_batch_keys_locate(batches, ctx: Context = None, weights=None) -> list:
        """verify_batch_locate for many keys in ONE device pass (b2g_verify_batch_keys_locate): batches as verify_batch_keys
        takes them.  Returns one list of bools per batch, equal to verify_batch_locate on that batch with the same weights
        (groups of 64 start at each batch's first proof); an empty batch gives [].  Weights, argument checks and errors as
        verify_batch_keys."""
        return _verify_batch_keys('verify_batch_keys_locate', batches, ctx, weights, False, True)

    @staticmethod
    def verify_batch_keys_locate_compressed(batches, ctx: Context = None, weights=None) -> list:
        """verify_batch_keys_locate on compressed proofs (b2g_verify_batch_keys_locate_compressed), decoded on the device: a
        blob that does not decode is False, and each batch's verdicts equal verify_batch_locate_compressed on that batch.
        Arguments, weights and errors as verify_batch_keys_locate; a blob that is not 128 bytes raises ValueError."""
        return _verify_batch_keys('verify_batch_keys_locate_compressed', batches, ctx, weights, True, True)

    # ---- compressed proofs: Proof::<Bn254>::serialize_compressed (ethereum.serialize_compressed), decoded on the device
    @staticmethod
    def decompress_proofs(blobs, ctx: Context = None) -> list:
        """Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5, Validate::Yes) for many proofs in one device pass
        (b2g_proofs_decompress): blobs = 128-byte bytes each.  Returns [Proof | None]: None where arkworks would refuse the
        blob (both flag bits set, a coordinate >= p, an x without a y, or a B outside G2).  A blob of another length raises
        ValueError."""
        blobs = list(blobs)
        rows = _proof_rows('decompress_proofs', blobs, True)
        if not blobs:
            return []
        ctx = ctx or default_context()
        data = np.frombuffer(rows, dtype=np.uint8).copy()
        out = np.zeros((len(blobs), 256), dtype=np.uint8)
        ok = np.zeros(len(blobs), dtype=np.uint8)
        N.check(N.lib().b2g_proofs_decompress(ctx._h, len(blobs), _ptr(data), _ptr(out), _ptr(ok)))
        return [Proof(row.tobytes()) if k else None for row, k in zip(out, ok)]

    @staticmethod
    def verify_many_compressed(vk, public_inputs, blobs, ctx: Context = None) -> list:
        """verify_many on compressed proofs (b2g_verify_many_compressed), decoded on the device: a verdict is True exactly
        when the blob decodes as decompress_proofs decodes it (G2 check of B included) and the decoded proof passes
        verify_many.  Arguments and errors as verify_many; a blob that is not 128 bytes raises ValueError."""
        return _verify_one_key('verify_many_compressed', 'many', vk, public_inputs, blobs, ctx, True)

    @staticmethod
    def verify_batch_compressed(vk, public_inputs, blobs, ctx: Context = None, weights=None) -> bool:
        """verify_batch on compressed proofs (b2g_verify_batch_compressed), decoded on the device: True exactly when every
        blob decodes and verify_batch with the same weights is True on the decoded proofs.  Arguments, weights and errors as
        verify_batch; a blob that is not 128 bytes raises ValueError."""
        return _verify_one_key('verify_batch_compressed', 'batch', vk, public_inputs, blobs, ctx, True, weights)

    @staticmethod
    def verify_batch_locate_compressed(vk, public_inputs, blobs, ctx: Context = None, weights=None) -> list:
        """verify_batch_locate on compressed proofs (b2g_verify_batch_locate_compressed), decoded on the device: a blob that
        does not decode is False, and the other verdicts are those of verify_batch_locate on the decoded proofs.  Arguments,
        weights and errors as verify_batch; a blob that is not 128 bytes raises ValueError."""
        return _verify_one_key('verify_batch_locate_compressed', 'batch_locate', vk, public_inputs, blobs, ctx, True, weights)

    # ---- rerandomization: Groth16::rerandomize_proof (ark-groth16 0.5.0), on the device (b2g_rerandomize_many)
    @staticmethod
    def rerandomize_proof(vk, proof: Proof, rng, ctx: Context = None) -> Proof:
        """Groth16::rerandomize_proof(vk, proof, rng): a new proof of the same statement, statistically indistinguishable
        from a fresh honest proof and unlinkable to `proof`; no witness is needed.  The factors are drawn as arkworks draws
        them (r1 = Fr::rand, r2 = Fr::rand, both again while either is zero, with fr_rand's limb rule), then
            A' = r1^-1 A,  B' = r1 B + (r1 r2) delta_2,  C' = C + r2 A.
        `vk` is a VerifyingKey, PreparedVerifyingKey or ProvingKey (prepared on the device once and cached per object, as for
        verify_many).  Raises ValueError when the proof is malformed (a coordinate >= p or a point off its curve); B is not
        checked for membership in G2, as in arkworks."""
        out = Groth16.rerandomize_proofs(vk, [proof], ctx=ctx, factors=[_rerandomize_factors(rng)])[0]
        if out is None:
            raise ValueError("rerandomize_proof: the proof is malformed (a coordinate >= p or a point off its curve)")
        return out

    @staticmethod
    def rerandomize_proofs(vk, proofs, rng=None, ctx: Context = None, factors=None) -> list:
        """rerandomize_proof for many proofs of one key in ONE device pass (b2g_rerandomize_many).  Proof i's factors are
        drawn from `rng` in order, as rerandomize_proof called on each proof in turn would draw them; the default rng is
        secrets.SystemRandom().  `factors` = one (r1, r2) per proof, each in [1, r), replaces the draw (a factor out of
        range raises B2gError, B2G_E_INPUT).  Returns [Proof | None]: None in place of a malformed proof, whose neighbours
        are unaffected."""
        proofs = list(proofs)
        for p in proofs:
            if len(p.data) != 256:
                raise ValueError("rerandomize_proofs: a proof is 256 bytes")
        if factors is None:
            import secrets
            rng = rng or secrets.SystemRandom()
            factors = [_rerandomize_factors(rng) for _ in proofs]
        factors = [(int(r1), int(r2)) for r1, r2 in factors]
        if len(factors) != len(proofs):
            raise ValueError("rerandomize_proofs: one (r1, r2) per proof")
        for i, pair in enumerate(factors):
            for name, f in zip(('r1', 'r2'), pair):
                if not 0 < f < R_MOD:
                    raise N.B2gError(N.B2G_E_INPUT, f"factor {name} of proof {i} is not in [1, r)")
        if not proofs:
            return []
        ctx = ctx or default_context()
        vh = ctx.vk_handle(vk)
        rows = np.frombuffer(b''.join(p.data for p in proofs), dtype=np.uint8).copy()
        r1 = np.frombuffer(b''.join(f.to_bytes(32, 'little') for f, _ in factors), dtype=np.uint8).copy()
        r2 = np.frombuffer(b''.join(f.to_bytes(32, 'little') for _, f in factors), dtype=np.uint8).copy()
        out = np.zeros((len(proofs), 256), dtype=np.uint8)
        ok = np.zeros(len(proofs), dtype=np.uint8)
        N.check(N.lib().b2g_rerandomize_many(ctx._h, vh, len(proofs), _ptr(rows), _ptr(r1), _ptr(r2), _ptr(out), _ptr(ok)))
        return [Proof(row.tobytes()) if k else None for row, k in zip(out, ok)]

    # base-range sharded variant: every rank calls prove_partial, the 768-byte partials are all-gathered by the caller
    # (torch.distributed / NCCL), then every rank calls prove_finish and obtains the same proof.
    @staticmethod
    def prove_partial(pk: ProvingKey, matrices: ConstraintMatrices, full_assignment, ctx: Context, r=None, s=None,
                      reduction=CircomReduction) -> np.ndarray:
        """r, s are optional here: when given, the (r, s)-only scalar multiplications start alongside the MSMs.  reduction:
        the key's R1CSToQAP, as for create_proof_with_reduction_and_matrices (LibsnarkReduction needs matrices with C)."""
        w = _c(full_assignment)
        ph, mh = ctx.pk_handle(pk), ctx.mat_handle(matrices, pk.n_vars, reduction.ID)
        out = np.zeros(N.PARTIAL_BYTES, dtype=np.uint8)
        rr = _scalar_bytes(r) if r is not None else None
        ss = _scalar_bytes(s) if s is not None else None
        N.check(N.lib().b2g_prove_partial(ctx._h, ph, mh, _ptr(rr) if rr is not None else None, _ptr(ss) if ss is not None else None, _ptr(w), _ptr(out)))
        return out

    @staticmethod
    def prove_sharded_p2p(pk: ProvingKey, matrices: ConstraintMatrices, r, s, full_assignment, ctx: Context, reduction=CircomReduction) -> Proof:
        """Sharded proof whose exchange runs inside the kernels over NVLink peer memory (sharding.connect_p2p first)."""
        w = _c(full_assignment)
        ph, mh = ctx.pk_handle(pk), ctx.mat_handle(matrices, pk.n_vars, reduction.ID)
        rr, ss = _scalar_bytes(r), _scalar_bytes(s)
        out = np.zeros(256, dtype=np.uint8)
        N.check(N.lib().b2g_prove_sharded_p2p(ctx._h, ph, mh, _ptr(rr), _ptr(ss), _ptr(w), _ptr(out)))
        return Proof(out.tobytes())

    @staticmethod
    def prove_finish(pk: ProvingKey, partials: np.ndarray, r, s, ctx: Context) -> Proof:
        parts = np.ascontiguousarray(partials, dtype=np.uint8).reshape(-1, N.PARTIAL_BYTES)
        rr, ss = _scalar_bytes(r), _scalar_bytes(s)
        out = np.zeros(256, dtype=np.uint8)
        N.check(N.lib().b2g_prove_finish(ctx._h, ctx.pk_handle(pk), _ptr(parts), parts.shape[0], _ptr(rr), _ptr(ss), _ptr(out)))
        return Proof(out.tobytes())
