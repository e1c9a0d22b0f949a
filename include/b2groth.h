/* b2groth.h - C ABI of libb2groth.so, the H100-native (sm_90a CUDA) Groth16/BN254 prover hot path that stands in
 * for what ark-circom 0.5 obtains from ark-groth16 / ark-ec / ark-poly on the CPU.
 *
 * The reference (arkworks-rs/circom-compat) has no FFI; its extension points are Rust traits and generic functions.
 * Each entry point below names the reference interface it replaces (paths relative to /root/reference):
 *
 *   b2g_pk_load            <- the ProvingKey<Bn254> half of read_zkey()                    src/zkey.rs:53-60, 103-133
 *   b2g_matrices_load      <- the ConstraintMatrices<Fr> half of read_zkey()               src/zkey.rs:151-196
 *   b2g_witness_map        <- CircomReduction::witness_map_from_matrices                   src/circom/qap.rs:23-88
 *   b2g_prove              <- Groth16::<Bn254, CircomReduction>::create_proof_with_reduction_and_matrices
 *                             (call sites src/zkey.rs:903-912, benches/groth16.rs:52-61, 72-80; body = ark-groth16
 *                             0.5.0 create_proof_with_assignment, restated in SURVEY.md 3.4)
 *   b2g_msm_g1 / b2g_msm_g2<- VariableBaseMSM::msm_bigint (ark-ec 0.5.0) as used by that function
 *   b2g_ntt                <- Radix2EvaluationDomain::{fft,ifft}_in_place (ark-poly 0.5.0) as used at qap.rs:60-81
 *   b2g_prove_many         <- the same function called for many witnesses of one circuit, in one device pass
 *   b2g_prove_keys         <- the same function called for batches of witnesses under many keys, in one device pass
 *   b2g_prove_partial / b2g_prove_finish : the same proof split for base-range sharding over several GPUs
 *   b2g_vk_load            <- GrothBn::process_vk(&params.vk) (src/zkey.rs:868, 914): the prepared verifying key, on the device
 *   b2g_vk_load_many       <- the same for many keys in one device pass
 *   b2g_verify_many        <- GrothBn::verify_with_processed_vk(&pvk, &inputs, &proof) (src/zkey.rs:869-870, 915-916), called
 *                             for many proofs of one key in one device pass
 *   b2g_verify_batch       <- the same check for a whole batch at once, as one random linear combination of the proofs
 *   b2g_proofs_decompress  <- Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5, Validate::Yes), for many proofs
 *   b2g_verify_many_compressed / b2g_verify_batch_compressed <- deserialize_compressed followed by the two calls above
 *   b2g_verify_batch_locate (+ _compressed) <- GrothBn::verify_with_processed_vk for every proof of a batch, at about the
 *                             batch check's cost when few proofs are invalid
 *   b2g_verify_batch_keys (+ _compressed) <- b2g_verify_batch for many keys, one verdict per key, in one device pass
 *   b2g_verify_batch_keys_locate (+ _compressed) <- b2g_verify_batch_locate for many keys, one verdict per proof, in one
 *                             device pass
 *   b2g_rerandomize_many   <- Groth16::rerandomize_proof (ark-groth16 0.5.0) for many proofs of one key, in one device pass
 *   b2g_points_serialize / b2g_points_deserialize <- CanonicalSerialize / CanonicalDeserialize (ark-serialize 0.5,
 *                             Validate::Yes) of the G1 / G2 points of a ProvingKey<Bn254> or VerifyingKey<Bn254>
 *   b2g_setup              <- Groth16::generate_parameters_with_qap (ark-groth16 0.5), which
 *                             generate_random_parameters_with_reduction calls (tests/groth16.rs:25): a whole proving key
 *   b2g_setup_from_powers  <- snarkjs groth16 setup (zkey new): a proving key from a powers-of-tau ceremony
 *   b2g_delta_update / b2g_delta_update_check <- snarkjs zkey contribute / the delta checks of snarkjs zkey verify
 *   b2g_powers_check       <- the algebraic checks of snarkjs powersoftau verify
 *   b2g_powers_prepare / b2g_lagrange_check <- snarkjs powersoftau prepare phase2 / the check of its sections 12-15
 *   b2g_powers_contribute <- snarkjs powersoftau contribute
 *   b2g_setup_from_lagrange <- snarkjs groth16 setup from a prepared ceremony, with no point transforms
 *   b2g_setup_check        <- snarkjs zkey verify: a proving key against its circuit and powers-of-tau ceremony
 *   b2g_fixed_base_g1/g2  <- the batch fixed-base multiplications of that setup, for the standard generators only
 *   b2g_wasm_load / b2g_witness_calculate <- WitnessCalculator::new + calculate_witness (src/witness/witness_calculator.rs):
 *                             a circom 2 circuit's .wasm run on the device, one lane per witness, many witnesses per call
 *
 * Conventions
 *   - every function returns 0 (B2G_OK) or a negative error code; b2g_last_error() gives a thread-local message.
 *     No exception or unwinding ever crosses this boundary.
 *   - field elements are 32 bytes, little-endian.  "mont" = Montgomery form with R = 2^256 exactly as a .zkey stores
 *     points (src/zkey.rs:327-332) and as arkworks keeps Fp256 in memory; "canon" = the plain integer.
 *   - G1 affine = x||y (64 B, mont), G2 affine = x.c0||x.c1||y.c0||y.c1 (128 B, mont); all-zero bytes = infinity
 *     (src/zkey.rs:340-360).
 *   - host pointers are only read/written during the call; handles own all device memory.
 *   - one proof in flight per b2g_ctx (a ctx is not thread-safe); create one ctx per GPU.
 *   - there is no CPU fallback: without a CUDA device every call fails with B2G_E_DEVICE.
 */
#ifndef B2GROTH_H
#define B2GROTH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B2G_API __attribute__((visibility("default")))
#else
#define B2G_API
#endif

#define B2G_OK 0
#define B2G_E_DOMAIN (-1) /* evaluation domain too large: SynthesisError::PolynomialDegreeTooLarge (qap.rs:31,66) */
#define B2G_E_SHAPE (-2)  /* inconsistent sizes / null pointers */
#define B2G_E_DEVICE (-3) /* CUDA failure, or no CUDA device */
#define B2G_E_INPUT (-4)  /* malformed input data */

typedef struct b2g_ctx b2g_ctx;
typedef struct b2g_pk b2g_pk;
typedef struct b2g_mat b2g_mat;
typedef struct b2g_pk_group b2g_pk_group;
typedef struct b2g_vk b2g_vk;

/* Proving key as read_zkey() produces it (src/zkey.rs:121-130); every pointer is a HOST pointer. */
typedef struct {
    uint32_t n_vars;          /* zkey header nVars  (src/zkey.rs:303) */
    uint32_t n_public;        /* zkey header nPublic */
    uint32_t domain_size;     /* zkey header domainSize = number of H bases */
    uint32_t reserved;
    const void* alpha_g1;     /* 64 B  */
    const void* beta_g1;      /* 64 B  */
    const void* delta_g1;     /* 64 B  */
    const void* beta_g2;      /* 128 B */
    const void* delta_g2;     /* 128 B */
    const void* a_query;      /* n_vars G1                 zkey section 5 */
    const void* b_g1_query;   /* n_vars G1                 zkey section 6 */
    const void* b_g2_query;   /* n_vars G2                 zkey section 7 */
    const void* l_query;      /* n_vars - n_public - 1 G1  zkey section 8 */
    const void* h_query;      /* domain_size G1            zkey section 9 */
} b2g_pk_desc;

/* ConstraintMatrices<Fr> a and b (src/zkey.rs:181-193) in CSR form; c is empty on the zkey route.  Values mont. */
typedef struct {
    uint32_t num_constraints; /* m: rows kept (src/zkey.rs:171-175) */
    uint32_t num_inputs;      /* num_instance_variables = n_public + 1 (src/zkey.rs:182) */
    uint32_t n_vars;          /* length of the full assignment */
    uint32_t reduction;       /* B2G_REDUCTION_CIRCOM (0) or B2G_REDUCTION_LIBSNARK (1): which R1CSToQAP the handle serves */
    const uint32_t* a_rowptr; /* m + 1 */
    const uint32_t* a_col;
    const void* a_val;        /* nnz x 32 B mont */
    const uint32_t* b_rowptr;
    const uint32_t* b_col;
    const void* b_val;
    const uint32_t* c_rowptr; /* LibsnarkReduction only (the zkey route has no C matrix, src/zkey.rs:188-192); else NULL */
    const uint32_t* c_col;
    const void* c_val;
} b2g_mat_desc;

/* CircomReduction: snarkjs keys, H query of domain_size bases, h = (ab - c)(g w^j), g = omega_2n   (src/circom/qap.rs:23-88).
 * LibsnarkReduction: arkworks-generated keys (the default QAP of Groth16<Bn254>, tests/groth16.rs:9,25-35), H query of
 * domain_size - 1 bases [tau^i Z(tau)/delta], h = coefficients of (ab - c)/Z (ark-groth16 0.5.0 r1cs_to_qap.rs). */
#define B2G_REDUCTION_CIRCOM 0
#define B2G_REDUCTION_LIBSNARK 1

B2G_API const char* b2g_last_error(void);
B2G_API int b2g_version(void);
B2G_API int b2g_device_count(int* count);

/* One context per GPU.  shard_rank / shard_count partition every query's base range (rank r of R owns the r-th
 * contiguous slice); use 0 / 1 for a whole-proof context. */
B2G_API int b2g_ctx_create(int device, int shard_rank, int shard_count, b2g_ctx** out);
B2G_API int b2g_ctx_destroy(b2g_ctx* ctx);

/* Optional: allocate this context's per-proof scratch for (pk, mat) now (otherwise the first proof does it, which
 * synchronises the device - do it up front when several contexts share a device). */
B2G_API int b2g_ctx_prepare(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat);

B2G_API int b2g_pk_load(b2g_ctx* ctx, const b2g_pk_desc* desc, b2g_pk** out);
B2G_API int b2g_pk_free(b2g_pk* pk);
B2G_API int b2g_matrices_load(b2g_ctx* ctx, const b2g_mat_desc* desc, b2g_mat** out);
B2G_API int b2g_matrices_free(b2g_mat* mat);

/* h = witness map of the handle's reduction; w_mont = n_vars x 32 B (host); h_out = domain x 32 B mont, natural order (host). */
B2G_API int b2g_witness_map(b2g_ctx* ctx, b2g_mat* mat, const void* w_mont, void* h_out, uint32_t* domain_size_out);

/* 256-byte proof: A.x A.y B.x.c0 B.x.c1 B.y.c0 B.y.c1 C.x C.y, canon little-endian; infinity = zeros.
 * r, s canon (32 B each).  Requires shard_count == 1. */
B2G_API int b2g_prove(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont,
              uint8_t proof_out[256]);

/* The same call split in two so that ONE host thread can keep several proofs in flight (one b2g_ctx each): submit
 * enqueues the upload, the captured proof graph and the read-back and returns without waiting for the device (w_mont
 * should be page-locked, or the upload is synchronous); wait blocks until that proof is done and fills the proof_out
 * given to submit, which must stay valid until then.  At most one proof may be pending per context.
 * b2g_prove == submit + wait.  (Reference shape: a rayon/thread pool calling the synchronous prove; here the pipeline is
 * a property of the device queue, not of host threads.) */
B2G_API int b2g_prove_submit(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont,
                             uint8_t proof_out[256]);
B2G_API int b2g_prove_wait(b2g_ctx* ctx);

/* b2g_prove_many <- the same Groth16::<Bn254, CircomReduction>::create_proof_with_reduction_and_matrices as b2g_prove, called
 * for many witnesses of one circuit (a caller's loop over that function).
 * count proofs for one (pk, mat) in one device pass: r_canon / s_canon = count x 32 B, w_mont = count pointers to n_vars x
 * 32 B full assignments, proofs_out = count x 256 B.  proofs_out[i] is byte-identical to b2g_prove with (r_i, s_i, w_i).
 * Synchronous.  Requires shard_count == 1 and 1 <= count <= 65535.  Every MSM sorts the whole batch into one list whose
 * bucket key is (proof, bucket), so each kernel of the pipeline runs once per batch with count times the parallelism, and
 * the latency-bound tails (fold, weighted bucket sum, glue) are paid once per batch.  The context's buffers grow to the
 * largest batch seen and are kept; DESIGN.md lists the device memory per batched proof and the largest count per size.
 * Errors: B2G_E_SHAPE for count == 0, null pointers, a sharded context, a shape mismatch, or count x bases x windows of a
 * query >= 2^32 (checked before anything is allocated); B2G_E_DEVICE when the batch's buffers do not fit in device memory.
 * It is the faster route up to 2^16 domains (H100 at 400 W: 2.3x three contexts in flight on the 2^14 bench key at count
 * 64, 1.1x at 2^16); from 2^18 up, where one proof fills the GPU, several contexts in flight are faster (README.md). */
B2G_API int b2g_prove_many(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, uint32_t count, const void* r_canon, const void* s_canon,
                           const void* const* w_mont, uint8_t* proofs_out);
/* b2g_prove_keys <- a caller's loop over Groth16::<Bn254, QAP>::create_proof_with_reduction_and_matrices for several keys
 * (circuits), e.g. a prover service whose queue mixes deposit, transfer and withdraw circuits: batches of witnesses under
 * n_keys proving keys in one device pass.
 *
 * b2g_pk_group_load loads n_keys keys (descs as b2g_pk_load takes them) with their matrix handles (mats[k] belongs to key k and
 * must outlive the group; a key may appear several times).  For each query (H, L, A, B1, B2) the window tables of all keys
 * are built into ONE arena at ONE window size c, msm_pick_c of the largest base count of that query in the group; key k's
 * rows start at its own row offset.  Each key keeps its sparse-B compaction, glue constants and 8-bit window tables as
 * b2g_pk_load builds them.  Device memory per key: its tables at the group's c (nwin(c) x bases x 64 B per G1 query,
 * x 128 B for B2), 2.6 MB of glue tables, 704 B of constants and 4 B per real B base of a sparse key.  A small key in a
 * group with a large one is built and sorted at the large key's c, so its proofs get 2^(c-1) buckets each (DESIGN.md
 * section 4).
 * Errors: B2G_E_SHAPE before anything is allocated for n_keys == 0, null pointers, a sharded context, a key whose
 * header or matrices disagree (b2g_prove's shape checks; the message names the key), or a query whose arena reaches 2^31
 * rows (the sign bit of an entry word); B2G_E_INPUT for an off-curve point (naming the key); B2G_E_DEVICE when the arena
 * does not fit.  On any error everything built so far is freed.
 *
 * b2g_prove_keys proves counts[k] witnesses under key k for every k, synchronously.  r_canon / s_canon = total x 32 B and
 * w_mont = total pointers (n_vars of the key each), key after key; proofs_out = total x 256 B in the same order.  The
 * proofs of key k are byte-identical to b2g_prove_many(ctx, pk_k, mat_k, counts[k], ...) with the same (r, s) and
 * witnesses.  Requires an unsharded context with no pending proof; 1 <= total <= 65535 (a count may be 0); and for each
 * query, total proofs x bases x windows < 2^32 sorted entries over the whole call.  Errors as b2g_prove_many.  The pass is
 * captured once as a CUDA graph per (group, counts) and replayed; the context keeps its buffers for the largest call. */
B2G_API int b2g_pk_group_load(b2g_ctx* ctx, uint32_t n_keys, const b2g_pk_desc* pks, b2g_mat* const* mats, b2g_pk_group** out);
B2G_API int b2g_pk_group_free(b2g_pk_group* group);
B2G_API int b2g_prove_keys(b2g_ctx* ctx, b2g_pk_group* group, const uint32_t* counts, const void* r_canon, const void* s_canon,
                           const void* const* w_mont, uint8_t* proofs_out);
/* The host half of the two calls above, without a device: bases = n_keys x 5 base counts (H, L, A, B1, B2: the domain,
 * n_vars - 1 for L and A, n_vars - 1 or the real B bases of a sparse key for B1 and B2); c_out = the group's 5 window sizes;
 * row_out = n_keys x 5 first arena rows.  With counts (n_vars / n_dom = each key's witness length and matrices domain),
 * rows_out = 3 x total rows of 4 u64 [first scalar, first canonical slot, base count, arena row] for the H sort (scalars in
 * the call's h vectors), the W sort (w[1..], for L and A) and the B sort (the gathered B scalars, for B1 and B2).  Errors as
 * the two calls for the same shapes. */
B2G_API int b2g_pk_group_layout(uint32_t n_keys, const uint32_t* bases, const uint32_t* n_vars, const uint32_t* n_dom, const uint32_t* counts,
                                int32_t* c_out, uint32_t* row_out, uint64_t* rows_out);

/* Page-lock / release a host buffer (cudaHostRegister): a witness vector owned by the caller (a Rust Vec<Fr>, a std::vector)
 * uploads asynchronously and at full PCIe speed once registered.  Registering twice / unregistering an unknown pointer is not
 * an error. */
B2G_API int b2g_host_register(const void* ptr, size_t bytes);
B2G_API int b2g_host_unregister(const void* ptr);

/* Sharded proof.  partial_out (768 B, host or device-accessible host memory) = this rank's partial MSM results
 * [H, L, A, B1] as G1 XYZZ (128 B each) followed by B2 as G2 XYZZ (256 B), mont.  b2g_prove_finish folds
 * shard_count partials in rank order and assembles the proof; every rank obtains identical bytes. */
#define B2G_PARTIAL_BYTES 768
/* r_canon / s_canon may be NULL; when given, the (r, s)-only part of the proof assembly (r*delta, s*delta, ...) is
 * started here on a side stream so that b2g_prove_finish with the same (r, s) finds it done. */
B2G_API int b2g_prove_partial(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont,
                              void* partial_out);
B2G_API int b2g_prove_finish(b2g_ctx* ctx, b2g_pk* pk, const void* partials_all, int count, const void* r_canon,
                     const void* s_canon, uint8_t proof_out[256]);

/* Sharded proof with the exchange fused into the proof-assembly kernel (NVLink peer memory instead of a host-driven
 * collective).  Every rank owns an exchange arena in its HBM (two slots of a 1 KiB record - the 768-byte partial plus s*A_k and
 * r*B1_k - with an epoch word each, then room for one transformed vector of the split witness map); peers map it through CUDA
 * IPC.  b2g_prove_sharded_p2p runs the partial MSMs, publishes the record with a system-scope release of the epoch, and the
 * gather kernel acquires every peer's epoch and reads the records straight out of peer memory; the assembly folds them in rank
 * order.  The whole sharded proof, exchange included, is one captured CUDA graph (the epoch is a device-resident counter).
 * All ranks must call it for the same proof; every rank obtains identical bytes.
 *   b2g_p2p_export  : B2G_IPC_HANDLE_BYTES: the cudaIpcMemHandle_t of this context's exchange arena + its capacity
 *   b2g_p2p_import  : records of ALL ranks in rank order (count x B2G_IPC_HANDLE_BYTES; the own entry is ignored)
 * With >= 3 ranks the witness map is split as well (CircomReduction): ranks 0, 1, 2 each transform ONE of a, b, c into their
 * arena, and every rank forms its slice of h = a*b - c reading the three vectors from peer HBM inside the pointwise kernel.
 * The arena is sized when it is first needed (export / import / connect_local) for the largest domain the context has been
 * prepared for, so call b2g_ctx_prepare BEFORE wiring the peers; otherwise every rank computes the whole map itself. */
#define B2G_IPC_HANDLE_BYTES 80
B2G_API int b2g_p2p_export(b2g_ctx* ctx, void* handle_out);
B2G_API int b2g_p2p_import(b2g_ctx* ctx, const void* handles_all, int count);
/* same wiring for shard contexts that live in ONE process (IPC handles cannot be opened by their exporter): ctxs in rank order */
B2G_API int b2g_p2p_connect_local(b2g_ctx** ctxs, int count);
B2G_API int b2g_prove_sharded_p2p(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon,
                                  const void* w_mont, uint8_t proof_out[256]);

/* Verifying key as ark-groth16's VerifyingKey<Bn254> holds it (params.vk, src/zkey.rs:103-119); every pointer is a HOST
 * pointer, points are affine Montgomery with the conventions of b2g_pk_desc (all-zero = infinity). */
typedef struct {
    uint32_t n_public;        /* public inputs per proof */
    uint32_t reserved;
    const void* alpha_g1;     /* 64 B  */
    const void* beta_g2;      /* 128 B */
    const void* gamma_g2;     /* 128 B */
    const void* delta_g2;     /* 128 B */
    const void* gamma_abc_g1; /* (n_public + 1) G1 */
} b2g_vk_desc;

/* b2g_vk_load <- GrothBn::process_vk (src/zkey.rs:868, 914; ark-groth16 0.5.0 prepare_verifying_key).  Checks that every point
 * is on its curve (B2G_E_INPUT otherwise), computes e(alpha, beta) with the device pairing, the line coefficients of -gamma and
 * -delta for every Miller-loop step, and an 8-bit window table per gamma_abc_g1[i + 1] (510 KiB each).  Like b2g_pk, the key is
 * a device object any context of the same device can use. */
B2G_API int b2g_vk_load(b2g_ctx* ctx, const b2g_vk_desc* desc, b2g_vk** out);
/* b2g_vk_load_many <- process_vk for n_keys keys in one device pass, for nodes that see many circuits (rollup and bridge nodes,
 * aggregators, verification layers whose clients send their keys with their proofs).  descs = n_keys descriptors (host);
 * out = n_keys handles.  out[k] holds, byte for byte, the device state b2g_vk_load(ctx, &descs[k]) builds (the points,
 * e(alpha, beta), the lines of -gamma and -delta, the window tables, which of gamma and delta are at infinity), and every call
 * that takes a b2g_vk takes it.  The same desc may appear more than once; each occurrence gets its own handle.
 * Memory: one device allocation per call, carved into every key's arrays (256-byte aligned).  Each handle holds a reference to
 * it: b2g_vk_free frees the handles one at a time, in any order, and the last one frees the allocation.
 * Cost: four kernel launches and two synchronises, whatever n_keys and the public-input counts: the on-curve checks of every
 * point, e(alpha, beta) one key per thread, the lines two threads per key, and every window table of every key in one launch.
 * b2g_vk_load is this call with one key.
 * All or nothing: on any error no handle is created, out is not written and the context stays usable.  Errors: B2G_E_SHAPE for
 * n_keys == 0 or a null pointer or field (the message names the key); B2G_E_INPUT for a point off its curve (the message
 * names the lowest key that holds one, and the point as b2g_vk_load names it); B2G_E_DEVICE when the keys do not fit in device
 * memory. */
B2G_API int b2g_vk_load_many(b2g_ctx* ctx, uint32_t n_keys, const b2g_vk_desc* descs, b2g_vk** out);
B2G_API int b2g_vk_free(b2g_vk* vk);
/* e(alpha, beta) as the loaded key holds it (PreparedVerifyingKey::alpha_g1_beta_g2): 384 B, twelve Montgomery Fq in the
 * order c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1 (host pointer) */
B2G_API int b2g_vk_alpha_beta(b2g_vk* vk, void* out);

/* b2g_verify_many <- GrothBn::verify_with_processed_vk (src/zkey.rs:869-870, 915-916), for count proofs of one key in one device
 * pass.  public_inputs = count x n_public canonical 32 B scalars (may be NULL when n_public == 0); proofs = count x 256 B in the
 * layout b2g_prove writes (canonical, all-zero point = infinity); verdicts_out = count bytes, 1 = valid, 0 = invalid.
 * A proof is valid iff e(A, B) e(IC[0] + sum x_i IC[i + 1], -gamma) e(C, -delta) == e(alpha, beta), with the host verifier's
 * semantics: a point at infinity contributes 1 to the product, a point not on its curve makes the proof invalid, and so does a
 * coordinate >= p (arkworks cannot deserialise such a proof; the C++ mirror's single call throws there instead).  No G2
 * subgroup check beyond the host verifier's.  Synchronous.
 * Errors: B2G_E_SHAPE for count == 0, null pointers, a key of another device or a proof pending on the context; B2G_E_INPUT for
 * a public input >= r (checked before anything runs); B2G_E_DEVICE when the batch's buffers do not fit in device memory (the
 * context stays usable).  The context's buffers grow to the largest batch seen and are kept. */
B2G_API int b2g_verify_many(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs,
                            uint8_t* verdicts_out);

/* b2g_verify_batch: whether ALL count proofs are valid, from one random-linear-combination pairing check, for callers that
 * only need the batch's verdict (an aggregator, a rollup node, a bridge).  When it is 0, b2g_verify_batch_locate finds the
 * invalid proofs.
 * public_inputs and proofs are laid out as for b2g_verify_many; weights = count x 16 B little-endian 128-bit weights r_i;
 * *verdict_out = 1 or 0.  The verdict is 1 iff every coordinate is below p, every point is on its curve, every B_i not at
 * infinity lies in G2 (the order-r subgroup of the twist; a proof whose B is outside G2 makes the batch invalid), and
 *     prod_i e(r_i A_i, B_i) * e(sum_i r_i C_i, -delta) * e(s_0 IC[0] + sum_j s_j IC[j + 1], -gamma) == e(alpha, beta)^s_0
 * with s_0 = sum_i r_i and s_j = sum_i r_i x_ij (mod r).  A point at infinity contributes 1 to the product, or nothing to a
 * sum, as in b2g_verify_many.
 * Soundness: for given weights the verdict is deterministic.  If every proof is valid under b2g_verify_many and every B is in
 * G2, the verdict is always 1; otherwise it is 0 except with probability at most 1 / (2^128 - 1) over uniformly drawn nonzero
 * weights.  This holds only if the weights are drawn AFTER the proofs are fixed, from a source the prover cannot predict or
 * influence (a CSPRNG); with weights the prover knows, invalid proofs can be made to cancel.
 * Cost: per proof a one-pair Miller loop, two 128-bit G1 products and a G2 membership test; the prepared pairs, the final
 * exponentiation and the public-input products are paid once per batch.  No per-(proof, input) G1 records are allocated.
 * Synchronous.  Errors as b2g_verify_many (B2G_E_SHAPE for count == 0, null pointers, a key of another device or a pending
 * proof; B2G_E_INPUT for a public input >= r; B2G_E_DEVICE when the buffers do not fit), plus B2G_E_INPUT for a zero weight;
 * every error leaves the context usable. */
B2G_API int b2g_verify_batch(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs,
                             const void* weights, uint8_t* verdict_out);

/* Compressed proofs: the 128-byte form of Proof::<Bn254>::serialize_compressed (ark-serialize 0.5) that arkworks-based
 * systems store and send: A.x (32 B), B.x.c0 (32 B), B.x.c1 (32 B), C.x (32 B), little-endian, each point's flags in the top
 * two bits of its last byte (bit 7: y is the larger of {y, -y}; bit 6: infinity).  A proof decodes as
 * Proof::<Bn254>::deserialize_compressed (Validate::Yes) decodes it: both flag bits set, a value >= p with the flags masked
 * off (infinity flag or not), an x whose y^2 has no square root, or a B outside G2 make it undecodable.  An undecodable proof
 * is never an error: it is invalid.  The decoding runs on the device, one proof per thread (csrc/verify.cu restates the rules).
 *
 * b2g_proofs_decompress <- Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5, Validate::Yes) for count proofs in one
 * device pass.  compressed = count x 128 B; proofs_out = count x 256 B in the b2g_prove layout (a point at infinity = zeros);
 * ok_out = count bytes (1 decoded, 0 not; the row of an undecodable proof is 256 bytes of 0xFF, which b2g_verify_many reports
 * invalid).  Synchronous.  Errors: B2G_E_SHAPE for count == 0, null pointers or a proof pending on the context;
 * B2G_E_DEVICE when the buffers do not fit (the context stays usable). */
B2G_API int b2g_proofs_decompress(b2g_ctx* ctx, uint32_t count, const void* compressed, uint8_t* proofs_out, uint8_t* ok_out);
/* b2g_verify_many_compressed <- deserialize_compressed followed by GrothBn::verify_with_processed_vk (src/zkey.rs:869-870,
 * 915-916), for count proofs of one key; b2g_verify_many on compressed proofs, decoded on the device without a round trip
 * through the host.  compressed = count x 128 B; the other arguments, the errors and the buffers as b2g_verify_many.  A verdict
 * is 1 exactly when the proof decodes (G2 check of B included) and the decoded proof passes b2g_verify_many. */
B2G_API int b2g_verify_many_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs,
                                       const void* compressed, uint8_t* verdicts_out);
/* b2g_verify_batch_compressed <- deserialize_compressed followed by the batch check of b2g_verify_batch.  compressed = count x
 * 128 B; the other arguments, the errors and the soundness statement as b2g_verify_batch.  The verdict is 1 exactly when every
 * proof decodes and b2g_verify_batch with the same weights gives 1 on the decoded rows. */
B2G_API int b2g_verify_batch_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs,
                                        const void* compressed, const void* weights, uint8_t* verdict_out);

/* Key points: the points of an arkworks-serialized ProvingKey<Bn254> / VerifyingKey<Bn254> (ark-groth16 0.5), for callers
 * that load or store such keys; the lengths and field order of the keys are parsed on the host (ark_serialize.py).  A
 * compressed point follows the rules of the compressed proofs above: G1 = x (32 B), G2 = x.c0, x.c1 (64 B), flags on the
 * last byte of x (of x.c1).  An uncompressed point is G1 = x, y (64 B) or G2 = x.c0, x.c1, y.c0, y.c1 (128 B), flags on the
 * last byte of y (of y.c1); bit 7 is written for the larger y and ignored on read.  A point at infinity is written as zero
 * coordinates with bit 6 set.  Both calls work in slices of a fixed number of points through one device buffer, so a key of
 * any size needs a bounded amount of device memory; they are synchronous, and every error leaves the context usable.
 *
 * b2g_points_serialize <- G1Affine / G2Affine::serialize_with_mode (ark-ec 0.5, CanonicalSerialize) for n points.  g2 = 0:
 * G1, 1: G2; compress = 0 or 1.  points_mont = n x 64 / 128 B (the b2g_pk_desc layout, all-zero = infinity); out = n x 32 /
 * 64 B (compressed) or 64 / 128 B (uncompressed).  Errors: B2G_E_SHAPE for null pointers or a proof pending on the context;
 * B2G_E_INPUT for a coordinate >= p (the message names the lowest such point); B2G_E_DEVICE when the buffer does not fit.
 *
 * b2g_points_deserialize <- G1Affine / G2Affine::deserialize_with_mode (ark-ec 0.5, CanonicalDeserialize, Validate::Yes) for
 * n points without any length prefix.  in = n points of the form above; points_out = n x 64 / 128 B Montgomery (all-zero =
 * infinity).  A point does not decode when both flag bits are set, a coordinate with its flags masked off is >= p (with the
 * infinity flag too), a compressed x has no y, an uncompressed point without the infinity flag is off its curve, or a G2
 * point not at infinity lies outside the order-r subgroup (G1 has cofactor 1).  *first_bad_out = the index of the lowest
 * point that does not decode, or n; such a point is not an error code.  points_out[i] is defined for i < *first_bad_out.
 * Errors: B2G_E_SHAPE for null pointers or a proof pending on the context; B2G_E_DEVICE when the buffer does not fit. */
B2G_API int b2g_points_serialize(b2g_ctx* ctx, int g2, int compress, size_t n, const void* points_mont, void* out);
B2G_API int b2g_points_deserialize(b2g_ctx* ctx, int g2, int compress, size_t n, const void* in, void* points_out,
                                   uint64_t* first_bad_out);

/* b2g_verify_batch_locate: one verdict per proof at about the cost of b2g_verify_batch when few proofs are invalid, for callers
 * that take proofs from untrusted submitters and must find the invalid ones.  The arguments, their layouts and the buffers are
 * those of b2g_verify_batch, except that verdicts_out = count bytes.
 * Proofs are split into groups of 64 consecutive proofs (the last group may be shorter).  Proof i is well-formed when every
 * coordinate is below p, every point is on its curve, and B is at infinity or lies in G2.  Its verdict is
 *   0 if it is not well-formed;
 *   else 1 if its group passes the batch equation of b2g_verify_batch taken over the group's well-formed proofs only, with the
 *     caller's weights for them (malformed proofs are left out of the product, of the sums and of s_0, s_j; a group without a
 *     well-formed proof has nothing left to check);
 *   else the b2g_verify_many verdict of the proof (the well-formed proofs of every failing group go through b2g_verify_many's
 *     kernels in one more device pass).
 * Completeness: a proof that b2g_verify_many accepts and whose B is in G2 always gets 1.
 * Soundness: any other proof gets 0, except with probability at most (the number of groups holding such a proof) / (2^128 - 1)
 * over uniformly drawn nonzero weights.  As for b2g_verify_batch, the weights must be drawn AFTER the proofs are fixed, from a
 * source the prover cannot predict or influence.
 * Determinism: for given weights the verdicts are deterministic.
 * Relation to b2g_verify_batch: every verdict is 1 exactly when b2g_verify_batch with the same weights gives 1, except in the
 * same low-probability event.  The two are not equal bit for bit: weights that make invalid proofs of different groups cancel
 * in the whole batch's equation do not make them cancel in their groups' equations.
 * Cost: b2g_verify_batch's per-proof work, plus per group one two-pair Miller loop, one final exponentiation, e(alpha, beta)^s_0
 * and the public-input products; plus b2g_verify_many on the well-formed proofs of the groups that fail.
 * Synchronous.  Errors as b2g_verify_batch: B2G_E_SHAPE for count == 0, null pointers, a key of another device or a pending
 * proof; B2G_E_INPUT for a public input >= r or a zero weight; B2G_E_DEVICE when the buffers do not fit.  Every error leaves
 * the context usable. */
B2G_API int b2g_verify_batch_locate(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs,
                                    const void* weights, uint8_t* verdicts_out);
/* b2g_verify_batch_locate_compressed: b2g_verify_batch_locate on compressed proofs, decoded on the device.  compressed = count x
 * 128 B; the other arguments, the rules and the errors as b2g_verify_batch_locate, where a proof that does not decode is not
 * well-formed.  The verdicts equal those of b2g_proofs_decompress followed by b2g_verify_batch_locate on the decoded rows. */
B2G_API int b2g_verify_batch_locate_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs,
                                               const void* compressed, const void* weights, uint8_t* verdicts_out);

/* One batch of proofs under one verifying key, for b2g_verify_batch_keys and b2g_verify_batch_keys_locate. */
typedef struct {
    b2g_vk* vk;
    uint32_t count;              /* proofs under this key (0 allowed) */
    uint32_t reserved;
    const void* public_inputs;   /* count x vk's n_public canonical 32 B scalars (NULL when n_public == 0 or count == 0) */
    const void* proofs;          /* count x 256 B (b2g_prove layout), or count x 128 B for the _compressed form */
    const void* weights;         /* count x 16 B nonzero 128-bit weights */
} b2g_key_batch;

/* b2g_verify_batch_keys: b2g_verify_batch for n_keys batches, each under its own key, in one device pass, for callers that
 * see many circuits with a few to a few hundred proofs each (rollup and bridge nodes, aggregators).  verdicts_out = n_keys
 * bytes.  verdicts_out[k] equals, bit for bit, *verdict_out of b2g_verify_batch(batches[k].vk, batches[k].count, the same
 * public inputs, proofs and weights): 1 iff every proof of batch k is well-formed (coordinates below p, points on their
 * curves, B at infinity or in G2) and batch k's equation of b2g_verify_batch holds.  A batch with count == 0 gets 1.  The
 * batches are independent: an invalid proof of batch k changes verdicts_out[k] only.  Each verdict keeps b2g_verify_batch's
 * soundness statement, with weights drawn after the proofs are fixed.  The same key may appear in several batches.
 * Cost: b2g_verify_batch's per-proof work over all proofs, plus per batch one two-pair Miller loop, e(alpha, beta)^s_0, one
 * final exponentiation and the public-input products; one device pass whatever the number of keys.
 * Synchronous.  Errors as b2g_verify_batch, with the key index in the message: B2G_E_SHAPE for n_keys == 0, a total count of
 * 0, null pointers, a key of another device or a pending proof; B2G_E_INPUT for a public input >= r or a zero weight;
 * B2G_E_DEVICE when the buffers do not fit.  Every error leaves the context usable. */
B2G_API int b2g_verify_batch_keys(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out);
/* b2g_verify_batch_keys_compressed: b2g_verify_batch_keys on compressed proofs (128 B each), decoded on the device.  A proof
 * that does not decode is malformed: verdicts_out[k] equals b2g_proofs_decompress followed by b2g_verify_batch_keys. */
B2G_API int b2g_verify_batch_keys_compressed(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out);

/* b2g_verify_batch_keys_locate: b2g_verify_batch_locate for n_keys batches, each under its own key, in one device pass, for
 * callers that see many circuits and take their proofs from untrusted submitters (rollup and bridge nodes, aggregators).
 * verdicts_out = one byte per proof, sum of batches[k].count bytes in batch order: batch k's verdicts start at the sum of
 * count_j over j < k, and a batch with count == 0 has none.  Batch k's verdicts equal, bit for bit, verdicts_out of
 * b2g_verify_batch_locate(batches[k].vk, batches[k].count, the same public inputs, proofs and weights).  Groups never cross
 * keys: a batch's groups of 64 start at its first proof and its last group may be shorter.  The completeness, soundness and
 * determinism statements of b2g_verify_batch_locate hold per batch.  The same key may appear in several batches.
 * Cost: b2g_verify_batch's per-proof work over all proofs, plus per group one two-pair Miller loop, one final exponentiation,
 * e(alpha, beta)^s_0 and the public-input products; plus b2g_verify_many's work on the well-formed proofs of the failing
 * groups, all keys in one more device pass.  The number of kernel launches does not depend on n_keys or on how many keys
 * fail.
 * Synchronous.  Errors as b2g_verify_batch_keys, with the key index in the message: B2G_E_SHAPE for n_keys == 0, a total
 * count of 0 or above 2^32 - 1, null pointers, a key of another device or a pending proof; B2G_E_INPUT for a public input >= r
 * or a zero weight; B2G_E_DEVICE when the buffers do not fit.  Every error leaves the context usable. */
B2G_API int b2g_verify_batch_keys_locate(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out);
/* b2g_verify_batch_keys_locate_compressed: b2g_verify_batch_keys_locate on compressed proofs (128 B each), decoded on the
 * device.  A proof that does not decode is not well-formed: batch k's verdicts equal those of
 * b2g_verify_batch_locate_compressed on batch k alone. */
B2G_API int b2g_verify_batch_keys_locate_compressed(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches,
                                                    uint8_t* verdicts_out);

/* b2g_rerandomize_many <- Groth16::rerandomize_proof(vk, proof, rng) (ark-groth16 0.5.0, src/prover.rs) for count proofs in one
 * device pass, for callers that hand stored proofs out again (relayers, credential services): each output is a proof of the
 * same statement, statistically indistinguishable from a fresh honest proof and unlinkable to its input (BKSV20, eprint
 * 2020/811, theorem 3).  No witness is needed.  For proof i = (A, B, C) and its factors r1 = r1_canon[i], r2 = r2_canon[i]:
 *     A' = r1^-1 A,   B' = r1 B + (r1 r2) delta_2,   C' = C + r2 A       (delta_2 = the key's delta_g2, r1^-1 and r1 r2 mod r)
 * Points at infinity follow the group law: A = infinity gives A' = infinity and C' = C, C = -r2 A gives C' = infinity.  As in
 * arkworks, B is not checked for membership in G2: a B outside G2 is transformed like any other point.
 * proofs = count x 256 B in the layout b2g_prove writes; r1_canon, r2_canon = count x 32 B canonical factors, each in
 * [1, r); proofs_out = count x 256 B, canonical affine (all zeros = infinity); ok_out = count bytes.  Row i is well-formed when
 * every coordinate is below p and every point not at infinity lies on its curve (the rule of b2g_verify_many).  A malformed
 * row is not an error: ok_out[i] = 0 and its output row is 256 bytes of 0xFF, which b2g_verify_many reports invalid; the other
 * rows are unaffected.  ok_out[i] = 1 otherwise.  The key's memory is used as b2g_vk_load left it (delta_2 only).
 * Cost: per proof one Fr inversion, two 254-bit G1 products of A, one joint 254-bit G2 chain over B and delta_2, and three
 * conversions to affine; one kernel, one proof per thread.
 * Synchronous.  Errors (checked before anything runs): B2G_E_SHAPE for count == 0, null pointers, a key of another device or a
 * proof pending on the context; B2G_E_INPUT for a factor that is zero or >= r (the message names the proof); B2G_E_DEVICE when
 * the buffers do not fit.  Every error leaves the context usable.  The buffers are the context's verification buffers: they
 * grow to the largest batch seen and are kept. */
B2G_API int b2g_rerandomize_many(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* proofs, const void* r1_canon,
                                 const void* r2_canon, uint8_t* proofs_out, uint8_t* ok_out);

/* The toxic waste of one setup: alpha, beta, gamma, delta, tau are 32 B canonical scalars; g1 / g2 are the generators the key
 * is built on, affine Montgomery (64 B / 128 B), or NULL for the standard ones (G1 = (1, 2), G2 = src/zkey.rs:443-463). */
typedef struct {
    const void* alpha; const void* beta; const void* gamma; const void* delta; const void* tau;
    const void* g1;
    const void* g2;
} b2g_setup_secrets;

/* HOST buffers the caller sized, in the b2g_pk_desc layout (affine Montgomery, all-zero = infinity). */
typedef struct {
    void *alpha_g1, *beta_g1, *delta_g1;            /* 64 B each */
    void *beta_g2, *gamma_g2, *delta_g2;            /* 128 B each */
    void *gamma_abc_g1;                             /* num_inputs G1 */
    void *a_query, *b_g1_query;                     /* n_vars G1 */
    void *b_g2_query;                               /* n_vars G2 */
    void *l_query;                                  /* n_vars - num_inputs G1 (may be NULL when that is 0) */
    void *h_query;                                  /* n G1 (CircomReduction) or n - 1 (LibsnarkReduction) */
} b2g_setup_out;

/* b2g_setup <- Groth16::generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, g1, g2) (ark-groth16 0.5) with tau given
 * instead of drawn, i.e. the key generate_random_parameters_with_reduction makes (tests/groth16.rs:25).  The circuit is a
 * b2g_mat_desc as b2g_matrices_load reads it: m rows in CSR form with Montgomery values, without the public-input rows (the
 * setup appends them, as the witness map does); `reduction` selects the H query; the C matrix is required for both reductions
 * (it may have no nonzeros).  With n the least power of two >= m + num_inputs and L_i = L_i(tau) the Lagrange coefficients of
 * the domain of size n:
 *     a_j = sum_rows A[r][j] L_r (+ L_(m+j) for j < num_inputs), b_j and c_j likewise without the extra term,
 *     a_query[j] = a_j g1, b_g1_query[j] = b_j g1, b_g2_query[j] = b_j g2 (j < n_vars),
 *     gamma_abc_g1[j] = (beta a_j + alpha b_j + c_j) / gamma g1 (j < num_inputs), l_query[j - num_inputs] = the same / delta,
 *     alpha_g1 = alpha g1, beta_g1 = beta g1, delta_g1 = delta g1, beta_g2 = beta g2, gamma_g2 = gamma g2, delta_g2 = delta g2,
 *     h_query (LibsnarkReduction) = tau^i (tau^n - 1) / delta g1, i < n - 1,
 *     h_query (CircomReduction)   = the odd entries of the inverse NTT over 2n points of (tau^i / delta, i < 2n - 1, then 0),
 *                                   times g1 (CircomReduction::h_query_scalars, src/circom/qap.rs:90-105).
 * Every scalar is computed on the device: the Lagrange coefficients as one inverse NTT of the powers of tau, the column sums by
 * a radix sort of the nonzeros by column and a reduce-by-key (no column is summed by one thread), the points by fixed-base
 * multiplication from window tables of g1 and g2, in slices through bounded device buffers.  Every device buffer that held a
 * secret or a value derived from one is zeroed before it is freed, and so is the library's host copy of the secrets.
 * Synchronous.  Errors (every error leaves the context usable; the content of the output buffers is then unspecified):
 * B2G_E_SHAPE for null pointers or fields, a missing C matrix, num_inputs of 0 or above n_vars, row pointers that do not start
 * at 0 or that decrease, a column index >= n_vars, an unknown reduction or a proof pending on the context (the matrix checks and
 * their messages are b2g_matrices_load's); B2G_E_DOMAIN for n above 2^27 (LibsnarkReduction) or 2^26 (CircomReduction, whose H
 * query needs the domain of 2n points); B2G_E_INPUT for a secret >= r, gamma or delta equal to 0, a generator coordinate >= p,
 * a generator at infinity or off its curve, or a g2 outside G2; B2G_E_DEVICE when the buffers do not fit in device memory. */
B2G_API int b2g_setup(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_setup_secrets* secrets, b2g_setup_out* out);

/* The points of a powers-of-tau ceremony of size 2^log_size (phase 1 of a snarkjs setup, sections 2-6 of a .ptau file), HOST
 * arrays in the b2g_pk_desc layout (affine Montgomery, all-zero = infinity):
 *   tau_g1 = tau^i g1 (i < 2^(p+1) - 1), tau_g2 = tau^i g2, alpha_tau_g1 = alpha tau^i g1, beta_tau_g1 = beta tau^i g1
 *   (i < 2^p), beta_g2 = beta g2. */
typedef struct {
    uint32_t log_size;           /* p, at most 28 */
    uint32_t reserved;
    const void* tau_g1;
    const void* tau_g2;
    const void* alpha_tau_g1;
    const void* beta_tau_g1;
    const void* beta_g2;
} b2g_powers_desc;

/* b2g_setup_from_powers <- `snarkjs groth16 setup circuit.r1cs pot.ptau` (snarkjs zkey new): a proving key from a ceremony
 * whose tau, alpha and beta nobody knows, with gamma = delta = 1 as snarkjs sets them.  The circuit and `out` are those of
 * b2g_setup.  With n the least power of two >= m + num_inputs, the call needs n <= 2^log_size and reads only the first
 * 2n - 1 / n / n / n points of tau_g1 / tau_g2 / alpha_tau_g1 / beta_tau_g1, so any ceremony at least as large serves.  With
 * [L_r] = iNTT_n(tau_g1[0..n))_r (the inverse radix-2 transform over points, natural order, scaled by n^-1), and [L_r]_2,
 * [alpha L_r], [beta L_r] likewise from tau_g2, alpha_tau_g1, beta_tau_g1:
 *     a_query[j] = sum_r A[r][j] [L_r] (+ [L_(m+j)] for j < num_inputs), b_g1_query[j] / b_g2_query[j] the same over B with
 *     [L_r] / [L_r]_2, gamma_abc_g1[j] (j < num_inputs) and l_query[j - num_inputs] (the others) =
 *     sum_r (A[r][j] [beta L_r] + B[r][j] [alpha L_r] + C[r][j] [L_r]) (+ [beta L_(m+j)] for j < num_inputs),
 *     alpha_g1 = alpha_tau_g1[0], beta_g1 = beta_tau_g1[0], delta_g1 = tau_g1[0], beta_g2 = beta_g2,
 *     gamma_g2 = delta_g2 = tau_g2[0],
 *     h_query (LibsnarkReduction) = tau_g1[i + n] - tau_g1[i], i < n - 1,
 *     h_query (CircomReduction)   = the odd entries of the inverse transform over 2n points of (tau_g1[0..2n-1), infinity),
 *                                   computed as 1/2 iNTT_n(y), y_i = omega_2n^-i (tau_g1[i] - tau_g1[i + n]).
 * The key equals, byte for byte, b2g_setup(circuit, alpha, beta, gamma = 1, delta = 1, tau) on the generators g1 = tau_g1[0]
 * and g2 = tau_g2[0].  The call checks only what it reads: every point read lies on its curve with coordinates below p, the
 * G2 points are in G2, and tau_g1[0], tau_g2[0] are not at infinity.  Whether the arrays really are powers of one tau with
 * the same alpha and beta is checked by b2g_powers_check, which callers run first.
 * Cost: four inverse transforms over G1 and one over G2 of n points, each (n/2) log2 n variable-base products; one product
 * per nonzero (a coefficient k above r/2 multiplies the negated point by r - k, so +-1 and small constants are cheap).
 * Synchronous.  Errors (every error leaves the context usable): the matrix checks and messages of b2g_setup (B2G_E_SHAPE);
 * B2G_E_DOMAIN for n > 2^log_size or at b2g_setup's domain limits; B2G_E_INPUT for a point off its curve or with a coordinate
 * >= p, a G2 point outside G2, or tau_g1[0] / tau_g2[0] at infinity, naming the array and index ("tau_g2[17]: not in G2");
 * B2G_E_SHAPE for null pointers or a pending proof; B2G_E_DEVICE when the buffers do not fit in device memory. */
B2G_API int b2g_setup_from_powers(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers, b2g_setup_out* out);

/* The prepared Lagrange sections 12-15 of a ceremony prepared at power p = log_size (what `snarkjs powersoftau prepare phase2`
 * adds), HOST arrays in the b2g_pk_desc layout.  Block k of a section starts at point 2^k - 1 and holds iNTT_(2^k) of the first
 * 2^k points of its monomial array (natural order, scaled by 2^-k), so entry i is L_i(tau) times the base point over the domain
 * of 2^k points:
 *   tau_g1        blocks k = 0 .. p + 1 (2^(p+2) - 1 points); block p + 1 transforms (tau_g1[0 .. 2^(p+1) - 1), infinity)
 *   tau_g2, alpha_tau_g1, beta_tau_g1   blocks k = 0 .. p (2^(p+1) - 1 points each).
 * A call for a domain of 2^log_n points reads only blocks up to log_n (+ 1 for tau_g1): any prefix of whole blocks serves. */
typedef struct {
    uint32_t log_size;           /* p, at most 26 */
    uint32_t reserved;
    const void* tau_g1;
    const void* tau_g2;
    const void* alpha_tau_g1;
    const void* beta_tau_g1;
} b2g_lagrange_desc;

/* The output buffers of b2g_powers_prepare: sections 12-15 of a ceremony of power log_size, sized as b2g_lagrange_desc says. */
typedef struct {
    uint32_t log_size;
    uint32_t reserved;
    void* tau_g1;
    void* tau_g2;
    void* alpha_tau_g1;
    void* beta_tau_g1;
} b2g_lagrange_out;

/* b2g_powers_prepare <- `snarkjs powersoftau prepare phase2`: sections 12-15 of the ceremony of power K = out->log_size formed by
 * the prefix of `powers` (tau_g1[0 .. 2^(K+1) - 1), tau_g2 / alpha_tau_g1 / beta_tau_g1[0 .. 2^K)), 1 <= K <= min(log_size, 26),
 * written into the caller's host buffers (memory-mapped output files serve).  Block K + 1 of tau_g1 is padded with infinity
 * whatever the input's size, as a ceremony of power K has only 2^(K+1) - 1 powers; K is capped at 26 because that block is a
 * 2^27-point transform, the limit of b2g_points_intt.
 * Blocks of fewer than 2^16 points (all four sections) run as ONE segmented pass: one launch per round t, running stage
 * k - 1 - t of every block k that has one (one launch for the three G1 sections, one for G2), the twiddles of every block taken
 * from the largest small domain's table, then one segmented finish (bit-reverse, scale by 2^-k, affine) that writes each block
 * at its section offset.  Below 2^16 points a block's stage is under two waves of the GPU, so per-block launches would only
 * add latency; the launch count of these blocks is 2 x 15 + 4 whatever K is.  Larger blocks run the transform of
 * b2g_points_intt, one block at a time.
 * The call checks what it reads as b2g_setup_from_powers does: every point lies on its curve with coordinates below p, the G2
 * points are in G2, tau_g1[0] and tau_g2[0] are not at infinity.  Whether the powers are a ceremony is b2g_powers_check's
 * question.  Cost: per section, the transforms of all blocks, sum_k (2^k / 2) k variable-base products (about twice those of
 * the top block).  Device memory: about 2^(K+1) x 256 B for the top G1 block (its XYZZ work area, its affine points and its
 * domain's tables), about 40 MB for the segmented pass, and the output goes back through one 64 MiB pinned staging buffer.
 * Synchronous.  Errors (every error leaves the context usable; on error the output buffers hold unspecified bytes):
 * B2G_E_DOMAIN for K outside [1, min(log_size, 26)] or log_size > 28; B2G_E_INPUT for a point that breaks a rule, naming the
 * array and index ("tau_g2[17]: not in G2"); B2G_E_SHAPE for null pointers or a pending proof; B2G_E_DEVICE when the buffers do
 * not fit. */
B2G_API int b2g_powers_prepare(b2g_ctx* ctx, const b2g_powers_desc* powers, const b2g_lagrange_out* out);

/* b2g_setup_from_lagrange: b2g_setup_from_powers without its point transforms.  [L_r], [L_r]_2, [alpha L_r], [beta L_r] are
 * read from block log_n of the four Lagrange sections instead of transformed; the column sums, the public-input rows and the
 * LibsnarkReduction H query are those of b2g_setup_from_powers.  The CircomReduction H query is the odd entries of block
 * log_n + 1 of lagrange tau_g1, which transforms all 2n powers T_0 .. T_(2n-1) except at log_n = lagrange->log_size, where that
 * block is padded with infinity.  The key keeps b2g_setup_from_powers's (and the reference's) H, the transform of
 * (T_0 .. T_(2n-2), infinity), so below the prepared power the call subtracts the term of T_(2n-1):
 *     h_query[i] = B_(2i+1) - (2n)^-1 omega_2n^(2i+1) T_(2n-1)   (B: block log_n + 1),
 * n products of one point from an 8-bit window table.  tau_g1 must then hold 2n points (it is read at 2n - 1).
 * The key equals b2g_setup_from_powers's byte for byte when the Lagrange sections are the transforms of the powers, which
 * b2g_lagrange_check decides.  The call reads and checks the same monomial points as b2g_setup_from_powers, and the Lagrange
 * points it reads with the same rules (infinity allowed), naming them lagrange_tau_g1 .. lagrange_beta_tau_g1 with the index in
 * their section.  Errors: those of b2g_setup_from_powers, and B2G_E_DOMAIN for n > 2^lagrange->log_size or
 * lagrange->log_size > 26. */
B2G_API int b2g_setup_from_lagrange(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers,
                                    const b2g_lagrange_desc* lagrange, b2g_setup_out* out);

/* The verdict of b2g_powers_check and b2g_lagrange_check.  rule: 0 none (ok), 1 a coordinate >= p, 2 off its curve, 3 at
 * infinity, 4 outside G2, 5 not the generator, 6 the powers are not those of one tau, alpha and beta, 7 the Lagrange section
 * `array` is not the transform of its monomial array.  array (rules 1-5, 7): 0 tau_g1, 1 tau_g2, 2 alpha_tau_g1, 3 beta_tau_g1,
 * 4 beta_g2, 5 lagrange_tau_g1, 6 lagrange_tau_g2, 7 lagrange_alpha_tau_g1, 8 lagrange_beta_tau_g1; index: the point in that
 * array (its index in the section for 5-8). */
typedef struct {
    uint8_t ok;
    uint8_t rule;
    uint8_t array;
    uint8_t reserved[5];
    uint64_t index;
} b2g_powers_report;

/* b2g_powers_check <- the algebraic checks of `snarkjs powersoftau verify`: whether the prefix a domain of n = 2^log_n points
 * reads (1 <= log_n <= log_size <= 28) is a ceremony, checked in one streamed pass over the host arrays.  With T = tau_g1
 * (2n - 1 points), U = tau_g2 (n), A = alpha_tau_g1 (n), B = beta_tau_g1 (n) and beta_2 = beta_g2, out->ok = 1 iff
 *   the point rules hold: every point read has coordinates below p, lies on its curve and is not at infinity; every G2 point
 *   is in G2; T_0 = G1 = (1, 2) and U_0 = the standard G2 generator (ark-bn254, EIP-197);
 *   and the ratio rules hold, all at once through one random linear combination:
 *     e(T_(i+1), U_0) = e(T_i, U_1), i < 2n - 2;   e(A_(i+1), U_0) = e(A_i, U_1) and e(B_(i+1), U_0) = e(B_i, U_1), i < n - 1;
 *     e(T_0, U_(i+1)) = e(T_1, U_i), i < n - 1;     e(B_0, U_0) = e(T_0, beta_2).
 * challenges = 5 x 32 B canonical rho, sigma, pi, kappa, eps in [1, r).  With S_X = sum_(i < |X|) rho^i X_i (one tableless
 * MSM per array), the shifted sums are sum_(i < M-1) rho^i X_(i+1) = rho^-1 (S_X - X_0) and sum_(i < M-1) rho^i X_i =
 * S_X - rho^(M-1) X_(M-1), so that, multiplied through by rho, every equation above is one term of
 *     P_hi = (S_T - T_0) + sigma (S_A - A_0) + pi (S_B - B_0) + eps B_0,
 *     P_lo = rho [(S_T - rho^(2n-2) T_(2n-2)) + sigma (S_A - rho^(n-1) A_(n-1)) + pi (S_B - rho^(n-1) B_(n-1))],
 *     e(P_hi, U_0) e(-P_lo, U_1) e(kappa T_0, S_U - U_0) e(-kappa rho T_1, S_U - rho^(n-1) U_(n-1)) e(-eps T_0, beta_2) == 1,
 * each with its own monomial (rho^(i+1), sigma rho^(i+1), pi rho^(i+1), kappa rho^(i+1), eps).
 * Soundness, as for b2g_verify_batch: an honest ceremony always gives ok = 1.  Once the point rules hold every point lies in a
 * group of prime order r, so by Schwartz-Zippel a ceremony that breaks any ratio rule gives ok = 1 with probability at most
 * 2n / (r - 1) (about 2^-224 at log_n = 28), and only if the challenges are drawn uniformly from [1, r) AFTER the ceremony is
 * fixed, from a source its authors cannot predict or influence.
 * A failure names the first point in section order (tau_g1, tau_g2, alpha_tau_g1, beta_tau_g1, beta_g2; lowest index first)
 * that breaks a point rule, with the first rule it breaks in the order of the codes above; the pairing product (rule 6) is
 * evaluated only when every point passes.  The transcript of snarkjs (the BLAKE2b hash chain and the contributions' proofs of
 * knowledge) is not checked.
 * The arrays are read once, in slices of 2^22 points through pinned staging buffers, the copy of one slice overlapping the work
 * on the one before, so device memory does not grow with the ceremony.  Cost: one tableless MSM per array (about one mixed
 * addition per point and window), the G2 subgroup test per G2 point, and five Miller loops with one final exponentiation.
 * Synchronous.  Errors (every error leaves the context usable; a malformed point is a verdict, not an error): B2G_E_DOMAIN for
 * log_n outside [1, log_size] or log_size > 28; B2G_E_INPUT for a challenge that is 0 or >= r; B2G_E_SHAPE for null pointers or
 * a pending proof; B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_powers_check(b2g_ctx* ctx, const b2g_powers_desc* powers, uint32_t log_n, const void* challenges,
                             b2g_powers_report* out);

/* b2g_lagrange_check: whether blocks 0 .. log_n of the Lagrange sections 13-15 and blocks 0 .. log_n + 1 of section 12
 * (1 <= log_n <= lagrange->log_size <= 26) are the transforms of the monomial arrays of `powers`.  The transform matrix is
 * symmetric, so for weights w over a section's blocks
 *     sum_k sum_i w_(k,i) Lambda_(k,i) = sum_j s_j X_j,   s = sum_k pad(iNTT_(2^k)(w_k));
 * with w at global section index g equal to rho^g (rho 32 B canonical in [1, r)), the Lagrange side is one streamed MSM in the
 * powers-of-rho mode and the monomial side one in the explicit-scalar mode, s made once on the scalar NTT.  s is the same for
 * sections 13-15 (over 2^log_n monomials); section 12 adds its top block (2^(log_n+1) monomials, read from tau_g1, which must
 * then hold that many points), dropping the coefficient of the infinity that pads block p + 1 when log_n = p.  Each section
 * gives one equality of points, three in G1 and one in G2; no pairing.  out->ok = 1 iff the point rules hold on every Lagrange
 * point read (coordinates below p, on its curve, G2 points in G2; infinity allowed) and the four equalities hold.  The monomial
 * arrays are not checked: b2g_powers_check, which callers run first, does that.
 * Soundness: an honest file always gives ok = 1.  Once the point rules hold, a wrong section passes with probability at most
 * (its point count) / (r - 1), and only if rho is drawn uniformly from [1, r) AFTER the file is fixed.  Blocks above log_n are
 * not read.  A failure names the first failing point (section order, lowest index first), else the first failing section
 * (rule 7).  The sections are read as b2g_powers_check reads its arrays, once, in slices through pinned staging buffers;
 * device memory holds those buffers and 32 B x 12 x 2^log_n of scalars.  Cost: two tableless MSMs per section and log_n + 1
 * scalar transforms.
 * Synchronous.  Errors (every error leaves the context usable; a malformed point or a failed equality is a verdict): B2G_E_DOMAIN
 * for log_n outside [1, lagrange->log_size], lagrange->log_size > 26 or above powers->log_size; B2G_E_INPUT for rho 0 or >= r;
 * B2G_E_SHAPE for null pointers or a pending proof; B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_lagrange_check(b2g_ctx* ctx, const b2g_powers_desc* powers, const b2g_lagrange_desc* lagrange, uint32_t log_n,
                               const void* rho_canon, b2g_powers_report* out);

/* A whole proving key with its counts, HOST arrays in the b2g_pk_desc layout (affine Montgomery, all-zero = infinity).  An
 * array may be NULL when its count is 0. */
typedef struct {
    uint32_t n_vars;             /* points of a_query, b_g1_query and b_g2_query */
    uint32_t n_ic;               /* points of gamma_abc_g1 (num_inputs) */
    uint32_t n_l;                /* points of l_query */
    uint32_t n_h;                /* points of h_query */
    const void *alpha_g1, *beta_g1, *delta_g1;           /* 64 B each */
    const void *beta_g2, *gamma_g2, *delta_g2;           /* 128 B each */
    const void *gamma_abc_g1, *a_query, *b_g1_query, *b_g2_query, *l_query, *h_query;
} b2g_key_desc;

/* The verdict of b2g_setup_check.  rule: 0 none (ok); 1 a coordinate >= p, 2 off its curve, 3 at infinity, 4 outside G2 (the
 * point rules: side, field and index name the point); 6 the count of `field` is not the circuit's (index = the count the
 * circuit needs); 7 `field` is not the ceremony's point; 8 an equation fails (field: 7 a_query E1, 8 b_g1_query E2,
 * 9 b_g2_query E3, 6 gamma_abc_g1 / l_query E4, 11 h_query E5, 2 delta_g1 / delta_g2 E6).  side: 0 the key, 1 the ceremony.
 * field (side 0): 0 alpha_g1, 1 beta_g1, 2 delta_g1, 3 beta_g2, 4 gamma_g2, 5 delta_g2, 6 gamma_abc_g1, 7 a_query,
 * 8 b_g1_query, 9 b_g2_query, 10 l_query, 11 h_query; (side 1): b2g_powers_report's array codes. */
typedef struct {
    uint8_t ok;
    uint8_t rule;
    uint8_t side;
    uint8_t field;
    uint8_t reserved[4];
    uint64_t index;
} b2g_setup_report;

/* b2g_setup_check <- `snarkjs zkey verify circuit.r1cs pot.ptau circuit.zkey` without its transcript: whether `key` is the key
 * b2g_setup_from_powers makes from `circuit` and `powers`, followed by any chain of b2g_delta_update contributions.  The
 * circuit and the powers are those of b2g_setup_from_powers.  With n the domain, m the constraints, ni = num_inputs, N = n_vars,
 * A' = A with the public-input rows A'[m + j][j] = 1 (j < ni), T = tau_g1 (2n - 1 points), U = tau_g2, Al = alpha_tau_g1,
 * Be = beta_tau_g1 (n each), and [L_r] = iNTT_n(T)_r, the transform matrix is symmetric, so for column weights w
 *     sum_j w_j (sum_r M[r][j] [L_r]) = sum_k s_k T_k,   c = M w (by rows), s = iNTT_n(c) (a scalar transform).
 * challenges = 2 x 32 B canonical rho, sigma in [1, r); w_j = rho^j (j < N), v_i = sigma^i; s^A, s^B, s^C transform A'w, Bw,
 * Cw.  out->ok = 1 iff the counts are the circuit's (N, ni, N - ni, and n or n - 1 H points by the reduction); alpha_g1 = Al_0,
 * beta_g1 = Be_0, beta_g2 = the ceremony's beta_g2 and gamma_g2 = U_0, byte for byte; the point rules hold (the prefix of the
 * ceremony: b2g_setup_from_powers's rules; every key point: coordinates below p and on its curve, every G2 point in G2,
 * delta_g1 and delta_g2 not at infinity; query points may be at infinity); and, in this order,
 *     E1 sum_j w_j a_query[j] = sum_k s^A_k T_k          E2 sum_j w_j b_g1_query[j] = sum_k s^B_k T_k
 *     E3 sum_j w_j b_g2_query[j] = sum_k s^B_k U_k
 *     E4 e(sum_(j<ni) w_j IC_j, gamma_2) e(sum_(j>=ni) w_j L_(j-ni), delta_2) = e(sum_k (s^A_k Be_k + s^B_k Al_k + s^C_k T_k), U_0)
 *     E5 e(sum_i v_i H_i, delta_2) = e(sum_k h_k T_k, U_0), with, for CircomReduction, t = 1/2 iNTT_n(v),
 *        h_k = t_k omega_2n^-k (k < n), h_(k+n) = -t_k omega_2n^-k (k <= n - 2); for LibsnarkReduction h_k = -v_k (k < n - 1),
 *        h_(n-1) = 0, h_k = v_(k-n) (n <= k <= 2n - 2)
 *     E6 e(delta_1, U_0) = e(T_0, delta_2).
 * Soundness, as for b2g_powers_check: an honest key always gives ok = 1.  Once the point rules hold every point lies in a group
 * of prime order r, so by Schwartz-Zippel a key that breaks E1-E4 gives ok = 1 with probability at most (N - 1) / (r - 1), and
 * one that breaks E5 at most (n - 1) / (r - 1), and only if the challenges are drawn uniformly from [1, r) AFTER the key and
 * the ceremony are fixed, from a source their authors cannot predict or influence.  Whether the ceremony is one is
 * b2g_powers_check's question; E6 holds for any delta_2 = x U_0 with delta_1 = x T_0.
 * A failure reports the first failing check in the order above: counts, byte equalities, the ceremony's points (array order,
 * lowest index first), the key's points (field order), then E1-E6.  The key arrays and the ceremony prefix are read once from
 * host memory (memory-mapped files in place), in slices of 2^22 points through pinned staging buffers; device memory holds the
 * matrices and about 32 B x (N + 6n) of scalars, never the points.  Cost: one tableless MSM per array read, four over T, the
 * G2 subgroup test per G2 point, three scalar transforms of n points, and seven Miller loops with three final
 * exponentiations.  The transcript of snarkjs (zkey section 10, the contributions' hashes and proofs of knowledge) is not
 * checked.
 * Synchronous.  Errors (every error leaves the context usable; a malformed point, a wrong count or a failed equation is a
 * verdict, not an error): those of b2g_setup_from_powers for the circuit and the powers; B2G_E_INPUT for a challenge that is 0 or
 * >= r; B2G_E_SHAPE for null pointers or fields or a pending proof; B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_setup_check(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers, const b2g_key_desc* key,
                            const void* challenges, b2g_setup_report* report);

/* The part of a proving key a delta contribution changes, HOST buffers in the b2g_pk_desc layout. */
typedef struct {
    uint32_t n_l, n_h;           /* points of l_query and h_query */
    void* delta_g1;              /* 64 B */
    void* delta_g2;              /* 128 B */
    void* l_query;               /* n_l G1 (may be NULL when n_l == 0) */
    void* h_query;               /* n_h G1 (may be NULL when n_h == 0) */
} b2g_delta_key;

/* b2g_delta_update <- `snarkjs zkey contribute` (phase 2): one contribution with the secret x (32 B canonical, in [1, r)):
 *     after.delta_g1 = x before.delta_g1, after.delta_g2 = x before.delta_g2,
 *     after.l_query[i] = x^-1 before.l_query[i], after.h_query[i] = x^-1 before.h_query[i];
 * the other fields of the key are unchanged (the caller copies them).  A key from b2g_setup_from_powers given contributions
 * x_1, ..., x_k equals b2g_setup(..., gamma = 1, delta = x_1 ... x_k, tau) byte for byte.  x and x^-1 are handled as
 * b2g_setup handles its secrets: the library's host copy of x is wiped once it has reached the device, and every device
 * buffer that held x or x^-1 is zeroed before it is freed.  snarkjs's transcript (the proof of knowledge of x, the hashes of
 * zkey section 10) is not produced.
 * Synchronous.  Errors (every error leaves the context usable): B2G_E_SHAPE for null pointers, counts that differ between
 * before and after, or a pending proof; B2G_E_INPUT for x = 0 or x >= r, a point of `before` off its curve or with a
 * coordinate >= p, or before.delta_g2 outside G2 (naming the field and index); B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_delta_update(b2g_ctx* ctx, const b2g_delta_key* before, const void* x_canon, b2g_delta_key* after);

/* b2g_delta_update_check <- `snarkjs zkey verify`'s check of the delta contributions: whether `after` is `before` with one or
 * more contributions applied.  weights = (n_l + n_h) x 16 B nonzero 128-bit little-endian weights (rho_i for l_query, then
 * sigma_i for h_query).  *verdict_out = 1 iff
 *   the counts match; every point of `after` has coordinates below p and lies on its curve; after.delta_g1 and
 *   after.delta_g2 are not at infinity and after.delta_g2 is in G2; before.delta_g2 is not at infinity;
 *   e(delta_1', delta_2) = e(delta_1, delta_2');
 *   e(sum rho_i L'_i + sum sigma_i H'_i, delta_2') = e(sum rho_i L_i + sum sigma_i H_i, delta_2).
 * Soundness, as for b2g_verify_batch: an honest update (any chain of b2g_delta_update calls) always gives 1.  Any other
 * `after` gives 0, except with probability at most 1 / (2^128 - 1) per equation over uniformly drawn nonzero weights, and only
 * if the weights are drawn AFTER both keys are fixed, from a source the contributor cannot predict or influence.  The other
 * fields of the key are not read: the host compares them (both mirrors do).
 * Cost: two 128-bit G1 products per point, a tree of G1 sums, and four pairings.
 * Synchronous.  Errors (every error leaves the context usable): B2G_E_SHAPE for null pointers or a pending proof; B2G_E_INPUT
 * for a zero weight; B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_delta_update_check(b2g_ctx* ctx, const b2g_delta_key* before, const b2g_delta_key* after, const void* weights,
                                   uint8_t* verdict_out);

/* Kernel-level entry points (parity tests, benchmarks). All pointers host. */
B2G_API int b2g_msm_g1(b2g_ctx* ctx, const void* bases, const void* scalars, size_t n, int scalars_mont, void* out_xy_mont);
B2G_API int b2g_msm_g2(b2g_ctx* ctx, const void* bases, const void* scalars, size_t n, int scalars_mont, void* out_xy_mont);
B2G_API int b2g_ntt(b2g_ctx* ctx, void* data_mont, int log_n, int inverse);
B2G_API int b2g_fixed_base_g1(b2g_ctx* ctx, const void* scalars_canon, size_t n, void* out_affine_mont);
B2G_API int b2g_fixed_base_g2(b2g_ctx* ctx, const void* scalars_canon, size_t n, void* out_affine_mont);
/* b2g_points_intt: the inverse radix-2 transform over n = 2^log_n affine points (g2 = 0: G1, 1: G2), in place, natural order,
 * scaled by n^-1 as b2g_ntt scales it: out_k = n^-1 sum_i omega_n^(-ik) in_i (log_n in 1..27, else B2G_E_DOMAIN).  The points
 * are not checked.  The kernel b2g_setup_from_powers runs. */
B2G_API int b2g_points_intt(b2g_ctx* ctx, int g2, int log_n, void* points_mont);
/* b2g_powers_msm: sum_(i < n) rho^i P_i over n host affine points (g2 = 0: G1, 64 B each; 1: G2, 128 B), rho 32 B canonical
 * (below r, else B2G_E_INPUT), out 64 / 128 B affine Montgomery (all-zero = infinity).  The tableless streamed MSM
 * b2g_powers_check runs: the points are read once, in slices, and are not checked.  B2G_E_SHAPE for null pointers or a
 * pending proof; n = 0 gives infinity. */
B2G_API int b2g_powers_msm(b2g_ctx* ctx, int g2, size_t n, const void* bases, const void* rho_canon, void* out_affine);

/* b2g_points_scale: out_i = k_i P_i over n host affine points (g2 = 0: G1, 64 B each; 1: G2, 128 B), each with its own
 * canonical scalar k_i (scalars: n x 32 B little-endian, each below r, else B2G_E_INPUT naming the first that is not); out is
 * n affine Montgomery points in the same layout (all-zero = infinity), byte-equal to b2g_fixed_base_g1 / g2 of s_i k_i for
 * P_i = s_i G.  A point at infinity or k_i = 0 gives infinity.  G1 splits k = k1 + k2 lambda with |k1|, |k2| < 2^128 (GLV,
 * phi(x, y) = (beta x, y)); G2 splits k = k1 + k2 6x^2 with k1, k2 < 2^127 (GLS, psi the twist Frobenius, which acts as [6x^2]
 * only on G2: G2 points must be in G2, and, as for b2g_points_intt, the points are not checked).  Every lane runs the same 33
 * signed 4-bit windows over both halves (4 doublings, two additions from a table of 1..8 P per point).  The points are
 * streamed in slices of 2^22 through pinned staging buffers, so device memory does not grow with n.  Synchronous.  Errors:
 * B2G_E_SHAPE for null pointers or a pending proof; B2G_E_DEVICE when the buffers do not fit. */
B2G_API int b2g_points_scale(b2g_ctx* ctx, int g2, size_t n, const void* points, const void* scalars_canon, void* out);

/* The secrets of one phase-1 contribution: tau, alpha, beta, 32 B canonical each, in [1, r). */
typedef struct {
    const void* tau;
    const void* alpha;
    const void* beta;
} b2g_powers_secrets;

/* The output of b2g_powers_contribute: caller-owned HOST arrays with the counts of the input ceremony (2^(p+1) - 1 / 2^p /
 * 2^p / 2^p / 1 points), in the b2g_pk_desc layout; memory-mapped files serve.  None may overlap an input array. */
typedef struct {
    void* tau_g1;
    void* tau_g2;
    void* alpha_tau_g1;
    void* beta_tau_g1;
    void* beta_g2;
} b2g_powers_out;

/* b2g_powers_contribute <- `snarkjs powersoftau contribute` (phase 1): one contribution with the secrets (t, a, b) to the
 * whole ceremony `in` of power p = in->log_size (sections 2-6 of a .ptau: T = tau_g1, U = tau_g2, A = alpha_tau_g1,
 * B = beta_tau_g1, beta_2 = beta_g2):
 *     T'_i = t^i T_i (i < 2^(p+1) - 1),  U'_i = t^i U_i,  A'_i = a t^i A_i,  B'_i = b t^i B_i (i < 2^p),  beta_2' = b beta_2.
 * A ceremony of (tau, alpha, beta) becomes the ceremony of (tau t, alpha a, beta b).  The exponent of point i is its index in
 * the whole array.  Each array is streamed once in slices of 2^22 points: the scalars c t^i (c = 1, a or b) are made on the
 * device per slice, and each point is one b2g_points_scale product.  Cost: 2^(p+2) - 1 G1 and 2^p + 1 G2 variable-base
 * products (about 1.3 billion points at p = 28), plus the point rules.  The call checks every point it reads, as
 * b2g_powers_prepare does: coordinates below p, on its curve, not at infinity, tau_g1[0] and tau_g2[0] the standard generators,
 * every G2 point in G2 (which the G2 split needs); the first failure is refused naming the array and index
 * ("tau_g2[17]: not in G2").  The contribution is sound only if t, a and b are discarded: anyone who knows them can undo it.
 * The library's host copy of the secrets is wiped once it has reached the device, every device buffer that held them or the
 * per-point scalars (any two consecutive scalars give t) is zeroed before it is freed, on errors too, and nothing returns them.
 * snarkjs's transcript (section 7: the hash chain and the proofs of knowledge of t, a and b) is not produced.
 * Synchronous.  Errors (every error leaves the context usable; on error the output arrays hold unspecified bytes):
 * B2G_E_DOMAIN for log_size outside 1..28; B2G_E_INPUT for a secret that is 0 or >= r, or a point that breaks a rule;
 * B2G_E_SHAPE for null pointers, an output that overlaps the input, or a pending proof; B2G_E_DEVICE when the buffers do not
 * fit. */
B2G_API int b2g_powers_contribute(b2g_ctx* ctx, const b2g_powers_desc* in, const b2g_powers_secrets* secrets, const b2g_powers_out* out);

/* Element-wise device arithmetic, for unit parity tests of the field / group layers.
 * op: 0 fq_mul, 1 fq_add, 2 fq_sub, 3 fr_mul, 4 fr_add, 5 fr_sub, 6 fq_inv, 7 fr_inv (b ignored),
 *     8 g1_add (a, b, out = n x 64 B affine), 9 g2_add (n x 128 B), 10 g1_dbl, 11 g2_dbl (b ignored),
 *     12 g1 mixed add, 13 g2 mixed add, 14 fq_sqr, 15 fq a*b - b*b, 16 fq mul through the lazy-reduction blocks (32 B),
 *     17 fq2_mul, 18 fq2_sqr, 19 fq2 a*b - b*swap(a) (n x 64 B: c0 || c1).
 * Ops 20 and up take and return raw XYZZ records (X || Y || ZZ || ZZZ, Montgomery, infinity iff ZZ == 0; G1 128 B, G2 256 B)
 * and do not normalise the result:
 *     20 g1 add(a, b), 21 g1 madd(a, b = 64 B affine), 22 g1 dbl(a); 23 g2 add, 24 g2 madd (b = 128 B affine), 25 g2 dbl,
 *     26 one G2 lane-pair mixed addition (the G2 accumulation kernel's) onto record a of entry b,
 *     27 one lane pair folds a run of 16 entries (a = 16 x 160 B) from empty, out = the record as the two lanes store it;
 *        an entry is a 128 B affine point and a 32 B word whose bit 0 negates it,
 *     28 fq2 product as the G2 accumulation kernel inlines it (n x 64 B),
 *     29 fq plain 512-bit product a * b for a < 2^255 (a, b: 32 B; out: 64 B little-endian).
 * Ops 30 and up are the pairing tower (csrc/pairing.cuh) on Fq12 values of 12 x 32 B Montgomery, in the order
 * c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1 (out always 384 B):
 *     30 fq12 mul(a, b), 31 fq12 sqr, 32 cyclotomic sqr, 33 / 34 / 35 Frobenius a^p / a^(p^2) / a^(p^3),
 *     36 final exponentiation a^((p^12 - 1) / r), 37 pairing e(a, b) (a: 64 B G1 affine, b: 128 B G2 affine), 38 fq12 inverse,
 *     39 sparse line product a * (c0 + c3 w + c4 w^3) (b: c0 || c3 || c4, 3 x 64 B Fq2),
 *     40 Miller loop of the pair (a, b) without the final exponentiation (a: G1, b: G2 affine),
 *     41 / 42 one projective doubling / addition of b (G2 affine) step on the twist point a = X || Y || Z (3 x 64 B):
 *        out = the new X || Y || Z followed by the line's c0 || c1 || c2.
 * Ops 43-45 are the batch check's pieces:
 *     43 G2 membership of a (128 B G2 affine, on the twist): out = 8 B, 1 if a is in G2 (or infinity), else 0,
 *     44 r * a for a G1 affine a (64 B) and a 128-bit r (b: 16 B little-endian): out = 64 B affine,
 *     45 a^k for a cyclotomic Fq12 a and a canonical 256-bit k (b: 32 B): out = 384 B.
 * Ops 46-48 are the compressed-proof decoder's pieces (b ignored); each result is followed by a 32 B slot whose first 64-bit
 * word is 1 when there is a root / the point decodes, else 0:
 *     46 a square root of a (32 B Fq, mont): out = 64 B, the root (mont) then the slot,
 *     47 a square root of a (64 B Fq2, mont): out = 96 B,
 *     48 one compressed G2 point a (64 B: x.c0, then x.c1 with the flags) decoded without the G2 check: out = 160 B, the
 *        canonical affine point (zeros at infinity, 0xFF bytes when it does not decode) then the slot.
 * Ops 49-53 are the verifier's stages, each a launch of the kernel b2g_vk_load, b2g_verify_many or b2g_verify_batch runs
 * (b ignored unless stated; gamma and delta are G2 affine, 128 B, zeros = infinity, and their lines are those of -gamma and
 * -delta, prepared as b2g_vk_load prepares them):
 *     49 the Miller value of one verify_many proof record: a = 576 B, A (G1 64 B), B (G2 128 B), the prepared inputs and C
 *        (G1 64 B each), gamma, delta; a pair with a point at infinity contributes 1: out = 384 B,
 *     50 the prepared lines of -a for a G2 affine a (128 B, not infinity): out = 88 lines of c0 || c1 || c2 (88 x 192 B),
 *     51 x * P from the 8-bit window table of P as the public-input kernel computes it: a = x (32 B canonical), b = one G1
 *        affine P for all rows (64 B): out = 128 B XYZZ,
 *     52 the 8-bit window table of a G1 affine a (64 B): out = 32 x 255 affine points d * 256^w * a (w-major),
 *     53 the Miller value of verify_batch's two prepared pairs: a = 512 B, the prepared inputs and sum r C (G1 XYZZ, 128 B
 *        each), gamma, delta: out = 384 B.
 * Op 54 is b2g_points_scale's scalar decomposition (b ignored): a = k (32 B canonical, below r): out = 128 B, the G1 split
 *     k = k1 + k2 lambda (mod r), then the G2 split k = k1 + k2 6x^2, each half as 32 B little-endian two's complement.
 * Operand and result sizes per row therefore differ by op; b may be NULL where the op does not read it. */
B2G_API int b2g_test_op(b2g_ctx* ctx, int op, const void* a, const void* b, size_t n, void* out);

/* Timing of the last b2g_prove / b2g_prove_partial on this ctx, CUDA-event milliseconds:
 * [0] h2d witness, [1] witness map, [2] msm H, [3] msm L, [4] msm A, [5] msm B1, [6] msm B2, [7] glue + d2h,
 * [8] whole call (first event to last event).  With the captured proof graph (default) [1]..[6] read 0: the graph has no
 * interior events (B2G_GRAPH=0 in the environment at b2g_ctx_create restores direct launches and the per-phase times).
 * Host wall-clock milliseconds of the same call: [9] entry -> upload enqueued, [10] entry -> everything enqueued,
 * [11] time blocked in the final wait. */
B2G_API int b2g_last_timings(b2g_ctx* ctx, float out_ms[16]);

/* Benchmark helper: the device-resident part of a proof (witness already in HBM from the last b2g_prove call):
 * runs witness map + 5 MSMs + glue `iters` times and returns the average CUDA-event milliseconds.  iters < 0: enqueue
 * |iters| proofs and return without waiting (*avg_ms = 0): the caller synchronises the device and times the window itself,
 * which is how several contexts are measured over ONE common window. */
B2G_API int b2g_bench_device(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int iters, float* avg_ms);
/* One MSM alone on the main stream, `iters` times (query: 0 H, 1 L, 2 A, 3 B1, 4 B2): out_ms[0] = average CUDA-event
 * milliseconds of the whole MSM, out_ms[1] = of its bucket-accumulation kernel (the dominant kernel, for the roofline). */
B2G_API int b2g_bench_msm(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int query, int iters, float out_ms[2]);
/* number of kernel launches issued by this library (process-wide, all contexts) so far; a replayed proof graph counts the kernel
 * nodes it contains */
B2G_API int b2g_launch_count(b2g_ctx* ctx, uint64_t* count);

/* ---------------------------------------------------------------------------------------------- circom 2 witnesses
 * A module is decoded, validated and translated on the host into the device interpreter's fixed-width code.  It must
 * use only the integer subset of WebAssembly 1.0 (every i32/i64 numeric, comparison and conversion op, the sign
 * extension ops, integer loads and stores, memory.size / memory.grow, select, drop, locals, globals, block, loop, if,
 * br, br_if, br_table, return, call, call_indirect, unreachable, active data and element segments) and import nothing
 * but the four circom 2 runtime functions (runtime.exceptionHandler, printErrorMessage, writeBufferMessage,
 * showSharedRWMemory).  Anything else is refused with B2G_E_SHAPE and b2g_last_error() names the cause (the function
 * index and opcode, the import, the missing export).
 *
 * b2g_wasm_load additionally requires the circom 2 protocol exports, and runs one lane on the device to read the
 * field (getFieldNumLen32 must be 8 and getRawPrime BN254's r) and the sizes; a circom 1 module is refused.
 * b2g_wasm_load_module loads any module of the subset for b2g_wasm_run (no protocol, no probe). */
typedef struct b2g_wasm b2g_wasm;
typedef struct {
    uint32_t n32;            /* getFieldNumLen32 */
    uint32_t witness_size;   /* getWitnessSize */
    uint32_t input_size;     /* getInputSize */
    uint32_t version;        /* getVersion: the circom major version */
    uint32_t mem_pages;      /* initial linear memory, 64 KiB pages */
    uint32_t reserved[3];
} b2g_wasm_summary;
/* Per-lane limits, read with b2g_wasm_get_limits and changed with b2g_wasm_set_limits.  memory.grow past max_pages
 * returns -1; a call deeper than max_depth, or whose locals and operand stack do not fit in stack_slots 8-byte slots
 * (the module's globals come first and need globals + 8 at least, else the limits are refused), ends the lane with
 * B2G_WASM_STACK; a lane that runs more than `fuel` translated instructions ends with B2G_WASM_FUEL.  budget_bytes bounds
 * the device memory a call uses for lane state: the lanes run in chunks of whole warps that fit it (0 = half the free
 * device memory, at most 32 GiB); a call whose budget cannot hold one warp (32 lanes) is refused with B2G_E_SHAPE.
 * Chunking does not change any result.  Defaults, sized from the module at load: its initial pages + 5 (within its
 * declared maximum), 256, globals + 4096, 2^32, 0.  On an H100 one lane runs 1-5 M instructions/s, so the default fuel
 * lets a lane caught in an endless loop hold the call for roughly 14 to 65 minutes: lower it for untrusted modules. */
typedef struct {
    uint32_t max_pages, max_depth, stack_slots, reserved;
    uint64_t fuel, budget_bytes;
} b2g_wasm_limits;
/* lane statuses */
#define B2G_WASM_OK 0
#define B2G_WASM_UNREACHABLE 1     /* unreachable executed */
#define B2G_WASM_MEMORY 2          /* a load or store outside the lane's memory */
#define B2G_WASM_DIV_ZERO 3        /* integer division or remainder by zero */
#define B2G_WASM_OVERFLOW 4        /* div_s of the minimum by -1 */
#define B2G_WASM_STACK 5           /* call depth or stack slots exhausted */
#define B2G_WASM_FUEL 6            /* instruction budget exhausted */
#define B2G_WASM_INDIRECT 7        /* call_indirect of an empty or out-of-range element, or of the wrong type */
#define B2G_WASM_PROTOCOL 8        /* getWitnessSize disagreed with the size the load read */
#define B2G_WASM_EXCEPTION 0x100   /* + c: the circuit called runtime.exceptionHandler(c) (4 = assert failed, ...) */

B2G_API int b2g_wasm_load(b2g_ctx* ctx, const void* bytes, size_t len, b2g_wasm** out);
B2G_API int b2g_wasm_load_module(b2g_ctx* ctx, const void* bytes, size_t len, b2g_wasm** out);
B2G_API int b2g_wasm_free(b2g_wasm* wasm);
B2G_API int b2g_wasm_info(b2g_wasm* wasm, b2g_wasm_summary* out);
B2G_API int b2g_wasm_get_limits(b2g_wasm* wasm, b2g_wasm_limits* out);
B2G_API int b2g_wasm_set_limits(b2g_wasm* wasm, const b2g_wasm_limits* limits);
/* count witnesses of one circuit, one device lane each, with no host step between the calls of the circom 2 protocol:
 * init(sanity_check); for input k (FNV-1a 64 hash hashes[k], split into its high and low 32 bits) and each of its
 * counts[k] values i: 8 x writeSharedRWMemory(j, limb j), setInputSignal(msb, lsb, i); getWitnessSize; for each wire
 * i: getWitness(i) and 8 x readSharedRWMemory(j).  Every witness has the same inputs; values_canon holds count x
 * sum(counts) 32-byte canonical values (below r), witness-major, inputs in order.  w_mont_out receives count x
 * witness_size x 32 B in Montgomery form (b2g_prove_many's layout; all zeros for a lane that did not finish) and
 * status_out one B2G_WASM_* status per witness. */
B2G_API int b2g_witness_calculate(b2g_ctx* ctx, b2g_wasm* wasm, uint32_t count, uint32_t n_inputs, const uint64_t* hashes,
                                  const uint32_t* counts, const void* values_canon, int sanity_check, void* w_mont_out,
                                  uint32_t* status_out);
/* count lanes each call the exported function `name` with nargs (at most 3) arguments, lane i taking
 * args[i*nargs .. i*nargs+nargs) (i32 zero-extended, i64 as is); results[i] = its result (0 if it has none). */
B2G_API int b2g_wasm_run(b2g_ctx* ctx, b2g_wasm* wasm, const char* name, uint32_t count, uint32_t nargs,
                         const uint64_t* args, uint64_t* results, uint32_t* status_out);

#ifdef __cplusplus
}
#endif
#endif /* B2GROTH_H */
