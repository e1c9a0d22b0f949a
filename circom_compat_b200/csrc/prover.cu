// prover.cu - contexts, device-resident proving keys / matrices, the proof pipeline and the C ABI (include/b2groth.h).
//
// Pipeline of one proof = Groth16::create_proof_with_reduction_and_matrices (call sites /root/reference/src/zkey.rs:903-912,
// benches/groth16.rs:52-61; body restated in SURVEY.md 3.3/3.4):
//     stream 0: H2D witness -> sparse mat-vec -> iNTT/coset/NTT -> h (stays in HBM) -> MSM over h_query
//     streams 1..4: MSMs over l_query / a_query[1..] / b_g1_query[1..] / b_g2_query[1..] against the witness
//     streams 2, 3: s*msm_A, r*msm_B1 right behind those MSMs; side stream: r*delta1, s*delta2, K_C (the (r, s)-only terms)
//     stream 0: glue (A, B2 and C = K_C + s*msm_A + r*msm_B1 + msm_L + msm_H, three affine conversions) -> D2H 256 B
#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cstring>
#include <vector>
#include "../../include/b2groth.h"
#include "ec.cuh"
#include "msm.cuh"
#include "fixed.cuh"
#include "ntt.cuh"
#include "setup.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {

// from msm.cu
void msm_build_table(MsmPlan& plan, const void* bases_dev, uint32_t n, bool g2, cudaStream_t st);
void msm_free_table(MsmPlan& plan);
void msm_scratch_alloc(MsmScratch& s, uint32_t n, int nwin, uint32_t nbuckets, bool g2, bool with_sort, uint32_t count = 1);
void msm_sort(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, uint32_t n, bool scalars_mont, cudaStream_t st, uint32_t count = 1,
              uint32_t scalar_stride = 0);
void msm_accumulate(const MsmPlan& plan, const MsmScratch& sorted, MsmScratch& acc, cudaStream_t st);
void msm_scratch_free(MsmScratch& s);
void msm_run(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, uint32_t n, bool scalars_mont, cudaStream_t st, uint32_t count = 1,
             uint32_t scalar_stride = 0);
void msm_init_kernels();
void msm_validate_points(const void* pts_dev, uint32_t n, bool g2, cudaStream_t st, const char* what);

enum { Q_H = 0, Q_L = 1, Q_A = 2, Q_B1 = 3, Q_B2 = 4, NQ = 5 };
static const size_t PARTIAL_OFF[NQ] = {0, 128, 256, 384, 512};
constexpr size_t REC_BYTES = B2G_PARTIAL_BYTES + 256;  // device-side record of one proof (or rank): the public 768-byte partial + [s*A_k, r*B1_k]
constexpr uint32_t MAX_BATCH = 65535;                 // proofs per b2g_prove_many call: the batch is a grid dimension of the sort kernels

}  // namespace b2g

using namespace b2g;

// a pass captured as a CUDA graph: the executable, the key it was captured for and the launches one replay stands for
struct GraphSlot {
    cudaGraphExec_t exec = nullptr;
    std::vector<uint64_t> key;
    uint64_t launches = 0;
};
enum { G_PROOF = 0, G_P2P = 1, G_KEYS = 2, NG = 3 };

struct b2g_ctx {
    int device = 0, shard_rank = 0, shard_count = 1;
    cudaStream_t st[NQ] = {}, st_glue = nullptr;
    cudaEvent_t ev_w = nullptr, ev_sort = nullptr, ev_pre = nullptr, ev_fork = nullptr, ev_done[NQ] = {}, ev_t[20] = {};
    MsmScratch scratch[NQ];
    bool scratch_ok = false;
    // Per-proof buffers hold cap_batch proofs (b2g_prove_many; 1 until a batch needs more), proof j at j x its size
    uint32_t cap_batch = 1;
    uint8_t* d_partial = nullptr;        // REC_BYTES: the public partial [H, L, A, B1] G1 XYZZ + B2 G2 XYZZ (768 B), then [s*A, r*B1]
    uint8_t* d_partials_all = nullptr;   // up to 64 ranks x REC_BYTES
    uint8_t* d_proof = nullptr;          // 256 B
    uint8_t* d_pre = nullptr;            // glue precomputation: r*d1, K_C (G1 XYZZ) + s*d2 (G2 XYZZ)
    fe *d_w = nullptr, *d_a = nullptr, *d_b = nullptr, *d_c = nullptr, *d_h = nullptr;   // batch: assignments n_vars apart, vectors n apart
    fe* d_wb = nullptr; size_t cap_wb = 0;     // gathered scalars of a sparse B query (b2g_pk::d_bidx), b_compact apart
    cudaEvent_t ev_sortb = nullptr; bool scratch_bsort = false;
    size_t cap_w = 0, cap_n = 0;               // elements d_w / d_a.. hold
    float last_ms[16] = {};
    bool pre_valid = false; uint32_t pre_r[8] = {}, pre_s[8] = {};   // (r, s) whose glue_pre result sits in d_pre
    uint8_t *d_rs = nullptr, *h_rs = nullptr;  // r | s (canonical, 2 x 32 B): device copy read by the glue kernels, pinned staging
    uint8_t *h_proof = nullptr, *pending_out = nullptr;   // pinned landing slot of the proof bytes; caller's buffer of submitted proofs
    uint32_t pending_count = 0;                           // proofs pending_out receives
    // One proof's whole device pipeline (all streams, ~100 launches) captured once per (key, matrices) as a CUDA graph and
    // replayed with a single launch: the host cost of a proof drops from ~130 driver calls to a handful (B2G_GRAPH=0 disables)
    bool use_graph = true;
    // [G_PROOF] whole proof (or batch) and [G_P2P] sharded proof with the peer-memory exchange, each captured for (key uid,
    // matrices uid, buffer generation, batch count); [G_KEYS] the b2g_prove_keys pass, for (group uid, buffer generation,
    // counts of every key), in a slot of its own so that it does not evict the one-key graph
    GraphSlot graphs[NG];
    uint64_t alloc_gen = 1;                                    // bumped whenever a buffer the graphs point into is (re)allocated
    unsigned long long* d_epoch = nullptr;                     // exchange epoch (device-resident so that it survives graph replay)
    // peer-memory exchange (b2g_prove_sharded_p2p): own buffer + every rank's buffer as seen from this device
    uint8_t* d_xchg = nullptr;                 // exchange arena (layout at EVAL_OFF below); allocated when the context is wired to its peers
    size_t eval_cap = 0, eval_common = 0;      // field elements the own arena holds / the smallest arena among all ranks
    uint8_t** d_peer_ptrs = nullptr;           // device array [shard_count]
    void* peer_mapped[64] = {};                // cudaIpcOpenMemHandle results (to close)
    int peers_imported = 0;
    VerifyBufs* vbufs = nullptr;               // b2g_verify_many scratch (verify.cu), grown on demand
    // b2g_prove_keys: the per-proof rows of its three sorts and the key of every proof (rewritten by each call)
    uint8_t* d_keyed = nullptr; size_t cap_keyed = 0;
};

static std::atomic<uint64_t> g_next_uid{1};            // handles are told apart by uid, not by address (addresses get reused)

struct b2g_pk {
    uint64_t uid = g_next_uid++;
    int device = 0, shard_rank = 0, shard_count = 1;   // a key may be used by any ctx of the same device and shard
    uint32_t n_vars = 0, n_public = 0, domain = 0;
    MsmPlan plan[NQ];
    uint32_t lo[NQ] = {}, cnt[NQ] = {}, scalar_off[NQ] = {};
    uint8_t* d_consts = nullptr;         // G1: alpha, beta, delta, a_query[0], b_g1_query[0] (5 x 64) ; G2: beta, delta, b_g2_query[0] (3 x 128)
    void *d_tab_delta1 = nullptr, *d_tab_delta2 = nullptr;   // 8-bit window tables of delta_g1 / delta_g2 (32 x 255 affine points)
    void *d_tab_aa = nullptr, *d_tab_bb = nullptr;           // same for alpha_g1 + a_query[0] and beta_g1 + b_g1_query[0] (glue_pre: K_C)
    // Sparse B: real circom keys have b_g1/b_g2_query entries at infinity for every wire that never occurs in a B row.  When
    // fewer than 80 % of this shard's B bases are real points, B1 and B2 are built over the compacted set only: d_bidx[j] =
    // position (inside the shard's w[1..] range) of the j-th real base; the proof gathers those scalars and sorts them on their own
    uint32_t* d_bidx = nullptr;
    uint32_t b_compact = 0;
};

namespace b2g { struct KeyGlue; }

// K proving keys loaded for proving under all of them in one pass (b2g_pk_group_load).  Every query's tables of all keys lie
// in one arena built at one window size; key k's rows of query q start at row[q][k].  The per-key state a proof reads besides
// those tables - glue constants, their window tables, the sparse-B compaction - sits in a b2g_pk of its own whose plan[q]
// holds no table, only the key's base count of the query.
struct b2g_pk_group {
    uint64_t uid = g_next_uid++;
    int device = 0;
    std::vector<b2g_pk*> keys;
    std::vector<b2g_mat*> mats;                // the caller's matrices, one per key (not owned)
    MsmPlan plan[NQ];                          // per query: the group's c, nwin, nbuckets; table = the arena
    std::vector<uint32_t> row[NQ];
    KeyGlue* d_keys = nullptr;                 // per key: the four window tables of glue_pre
    const uint8_t** d_consts = nullptr;        // per key: its d_consts (glue_post)
    bool b_sparse = false;                     // some key's B query is compacted: B1 and B2 get a sort of their own
    const uint32_t** d_bidx = nullptr;         // per key: d_bidx, null for a dense B query
};

struct b2g_mat {
    uint64_t uid = g_next_uid++;
    int device = 0;
    uint32_t m = 0, num_inputs = 0, n_vars = 0, n = 0;
    int logn = 0;
    NttDomain dom;
    uint32_t *a_rowptr = nullptr, *a_col = nullptr, *b_rowptr = nullptr, *b_col = nullptr, *c_rowptr = nullptr, *c_col = nullptr;
    fe *a_val = nullptr, *b_val = nullptr, *c_val = nullptr;
    uint32_t reduction = B2G_REDUCTION_CIRCOM;
};

namespace b2g {

thread_local std::string g_last_error;

struct Scalar256 { uint32_t l[8]; };

CtxView ctx_view(b2g_ctx* ctx) { return {ctx->device, ctx->st[0], ctx->pending_out != nullptr, &ctx->vbufs}; }

CtxView ctx_idle(b2g_ctx* ctx) {
    const CtxView cv = ctx_view(ctx);
    if (cv.proof_pending) throw_error(B2G_E_SHAPE, "a submitted proof is still pending on this context: call b2g_prove_wait first");
    return cv;
}

// ------------------------------------------------------------------------------------------------ glue kernels
// pre[0] = r*delta1, pre[1] = K_C = (r*s)*delta1 + s*(alpha1 + a_query[0]) + r*(beta1 + b_g1_query[0]) (G1 XYZZ, 128 B
// each); then s*delta2 (G2 XYZZ, 256 B).  Every base here is fixed per key: its 8-bit window table is built at b2g_pk_load,
// so each product is 32 table look-ups and a 5-level tree inside one warp instead of a 254-step double-and-add on one
// thread.  K_C is what is left of C = s*A + r*B1 - rs*delta1 + L + H once the MSM results are taken out:
// C = K_C + s*msm_A + r*msm_B1 + msm_L + msm_H  (A = alpha + a0 + msm_A + r*delta1, B1 likewise).
// One CTA per proof of a batch: CTA j reads (r, s) at rs[2j], rs[2j + 1] and writes pre + j * PRE_BYTES.
constexpr size_t PRE_BYTES = 2 * 128 + 256;
// one proof's precomputation by one CTA of 160 threads: (r, s) at rs[0], rs[1], result at pre
__device__ __forceinline__ void glue_pre_one(const void* __restrict__ tab_d1, const void* __restrict__ tab_d2, const void* __restrict__ tab_aa,
                                             const void* __restrict__ tab_bb, const Scalar256* __restrict__ rs, uint8_t* __restrict__ pre) {
    __shared__ G1::Pt sh1[4][32];
    __shared__ G2::Pt sh2[32];
    __shared__ G1::Pt res[4];
    const Scalar256 r = rs[0], s = rs[1];
    const int warp = threadIdx.x >> 5;
    const bool lead = (threadIdx.x & 31) == 0;
    if (warp < 4) {
        // warp 0: r*d1   1: rs*d1   2: s*(alpha + a0)   3: r*(beta1 + b0)
        Scalar256 k = (warp == 0 || warp == 3) ? r : s;
        if (warp == 1) {
            fe rc, sc;                                   // Scalar256 is only 4-byte aligned: copy limb by limb
            #pragma unroll
            for (int i = 0; i < 8; i++) { rc.l[i] = r.l[i]; sc.l[i] = s.l[i]; }
            fe rm = Fr::from_canonical(rc), sm = Fr::from_canonical(sc);
            fe rs_ = Fr::to_canonical(Fr::mul(rm, sm));
            #pragma unroll
            for (int i = 0; i < 8; i++) k.l[i] = rs_.l[i];
        }
        const void* tab = warp < 2 ? tab_d1 : (warp == 2 ? tab_aa : tab_bb);
        G1::Pt p = warp_fixed_mul<G1, Fq>(tab, k.l, sh1[warp]);
        if (lead) { res[warp] = p; if (warp == 0) pt_store<Fq>(pre, 0, p); }
    } else {
        G2::Pt p = warp_fixed_mul<G2, Fq2>(tab_d2, s.l, sh2);
        if (lead) pt_store<Fq2>(pre + 2 * 128, 0, p);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        G1::Pt kc = res[1];
        G1::add(kc, res[2]);
        G1::add(kc, res[3]);
        pt_store<Fq>(pre, 1, kc);
    }
}

__global__ void __launch_bounds__(160) glue_pre_kernel(const void* __restrict__ tab_d1, const void* __restrict__ tab_d2, const void* __restrict__ tab_aa,
                                                       const void* __restrict__ tab_bb, const Scalar256* __restrict__ rs, uint8_t* __restrict__ pre) {
    glue_pre_one(tab_d1, tab_d2, tab_aa, tab_bb, rs + 2 * blockIdx.x, pre + (size_t)blockIdx.x * PRE_BYTES);
}

// out = k * p for one XYZZ point (the partial A / B1 MSM result of a rank) - in a whole proof issued on that MSM's own stream
// as soon as it finishes, so the two variable-base scalar multiplications of the proof overlap the longest MSM instead of
// following it.  CTA j: pt and out in record j (REC_BYTES apart), k at k + j * kstep (2 for the proofs of a batch, whose
// (r, s) pairs are 2 apart; 0 for the rank records of one proof, which share one (r, s)).
__global__ void scale_partial_kernel(const uint8_t* __restrict__ pt, const Scalar256* __restrict__ k, uint8_t* __restrict__ out, int kstep) {
    if (threadIdx.x != 0) return;
    pt += blockIdx.x * REC_BYTES; out += blockIdx.x * REC_BYTES; k += kstep * blockIdx.x;
    const Scalar256 kk = *k;
    G1::Pt p = pt_load<Fq>(pt, 0);
    pt_store<Fq>(out, 0, G1::mul_scalar(p, kk.l));       // k == 0 -> infinity (r == 0: B1 drops out, prover.rs)
}

__device__ __forceinline__ void store_canon(uint8_t* out, int slot, const fe& v) { fe_store(out + 32 * slot, Fq::to_canonical(v)); }

// partials = count records of REC_BYTES: the 768-byte partial [H, L, A, B1 (G1 XYZZ), B2 (G2 XYZZ)], then [s*A_k, r*B1_k]
// (G1 XYZZ, scale_partial_kernel).  Folds them in rank order and assembles the proof (ark-groth16 0.5.0
// create_proof_with_assignment).  No scalar multiplication is left here: A, B2 and C are three independent sums, converted
// to affine by three warps side by side.
// CTA j of a batch assembles proof j from its own `count` records, precomputation and 256-byte proof slot.
__global__ void glue_post_kernel(const uint8_t* __restrict__ partials, int count, const uint8_t* __restrict__ consts, const uint8_t* __restrict__ pre,
                                 uint8_t* __restrict__ proof) {
    partials += (size_t)blockIdx.x * count * REC_BYTES;
    pre += (size_t)blockIdx.x * PRE_BYTES;
    proof += (size_t)blockIdx.x * 256;
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) != 0) return;
    if (warp == 0) {
        // A = r*delta1 + a_query[0] + msm_A + alpha1
        G1::Pt acc = pt_load<Fq>(pre, 0);
        G1::madd(acc, aff_load<Fq>(consts, 3));
        for (int k = 0; k < count; k++) { G1::Pt q = pt_load<Fq>(partials + (size_t)k * REC_BYTES + 256, 0); G1::add(acc, q); }
        G1::madd(acc, aff_load<Fq>(consts, 0));
        G1::Aff a = G1::to_affine(acc);
        store_canon(proof, 0, a.x); store_canon(proof, 1, a.y);
    } else if (warp == 1) {
        // C = K_C + sum_k (s*A_k + r*B1_k + L_k + H_k)
        G1::Pt acc = pt_load<Fq>(pre, 1);
        for (int k = 0; k < count; k++) {
            const uint8_t* rec = partials + (size_t)k * REC_BYTES;
            G1::Pt q = pt_load<Fq>(rec + B2G_PARTIAL_BYTES, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec + B2G_PARTIAL_BYTES + 128, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec + 128, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec, 0); G1::add(acc, q);
        }
        G1::Aff c = G1::to_affine(acc);
        store_canon(proof, 6, c.x); store_canon(proof, 7, c.y);
    } else {
        // B2 = s*delta2 + b_g2_query[0] + msm_B2 + beta2
        G2::Pt acc = pt_load<Fq2>(pre + 2 * 128, 0);
        G2::madd(acc, aff_load<Fq2>(consts + 5 * 64, 2));
        for (int k = 0; k < count; k++) { G2::Pt q = pt_load<Fq2>(partials + (size_t)k * REC_BYTES + 512, 0); G2::add(acc, q); }
        G2::madd(acc, aff_load<Fq2>(consts + 5 * 64, 0));
        G2::Aff b = G2::to_affine(acc);
        store_canon(proof, 2, b.x.c0); store_canon(proof, 3, b.x.c1); store_canon(proof, 4, b.y.c0); store_canon(proof, 5, b.y.c1);
    }
}

// ------------------------------------------------------------------------------------------------ keyed batches (b2g_prove_keys)
// The window tables of one key of a group that glue_pre_keys_kernel reads (b2g_pk_group::d_keys)
struct KeyGlue { const void *d1, *d2, *aa, *bb; };

// CTA j = proof j of a keyed batch: glue_pre_kernel with proof j's key's tables (key_of[j])
__global__ void __launch_bounds__(160) glue_pre_keys_kernel(const KeyGlue* __restrict__ keys, const uint32_t* __restrict__ key_of,
                                                            const Scalar256* __restrict__ rs, uint8_t* __restrict__ pre) {
    const KeyGlue k = keys[key_of[blockIdx.x]];
    glue_pre_one(k.d1, k.d2, k.aa, k.bb, rs + 2 * blockIdx.x, pre + (size_t)blockIdx.x * PRE_BYTES);
}

// CTA j = proof j of a keyed batch: glue_post_kernel's assembly from proof j's one record, with its key's constants
// (consts_of[key_of[j]]).  The body is glue_post_kernel's, restated rather than shared: sharing it changes the code
// ptxas makes for glue_post_kernel (a smaller stack frame), and the one-key kernel is left exactly as it was.
__global__ void glue_post_keys_kernel(const uint8_t* __restrict__ partials, const uint8_t* const* __restrict__ consts_of,
                                      const uint32_t* __restrict__ key_of, const uint8_t* __restrict__ pre, uint8_t* __restrict__ proof) {
    constexpr int count = 1;
    const uint8_t* __restrict__ consts = consts_of[key_of[blockIdx.x]];
    partials += (size_t)blockIdx.x * count * REC_BYTES;
    pre += (size_t)blockIdx.x * PRE_BYTES;
    proof += (size_t)blockIdx.x * 256;
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) != 0) return;
    if (warp == 0) {
        // A = r*delta1 + a_query[0] + msm_A + alpha1
        G1::Pt acc = pt_load<Fq>(pre, 0);
        G1::madd(acc, aff_load<Fq>(consts, 3));
        for (int k = 0; k < count; k++) { G1::Pt q = pt_load<Fq>(partials + (size_t)k * REC_BYTES + 256, 0); G1::add(acc, q); }
        G1::madd(acc, aff_load<Fq>(consts, 0));
        G1::Aff a = G1::to_affine(acc);
        store_canon(proof, 0, a.x); store_canon(proof, 1, a.y);
    } else if (warp == 1) {
        // C = K_C + sum_k (s*A_k + r*B1_k + L_k + H_k)
        G1::Pt acc = pt_load<Fq>(pre, 1);
        for (int k = 0; k < count; k++) {
            const uint8_t* rec = partials + (size_t)k * REC_BYTES;
            G1::Pt q = pt_load<Fq>(rec + B2G_PARTIAL_BYTES, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec + B2G_PARTIAL_BYTES + 128, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec + 128, 0); G1::add(acc, q);
            q = pt_load<Fq>(rec, 0); G1::add(acc, q);
        }
        G1::Aff c = G1::to_affine(acc);
        store_canon(proof, 6, c.x); store_canon(proof, 7, c.y);
    } else {
        // B2 = s*delta2 + b_g2_query[0] + msm_B2 + beta2
        G2::Pt acc = pt_load<Fq2>(pre + 2 * 128, 0);
        G2::madd(acc, aff_load<Fq2>(consts + 5 * 64, 2));
        for (int k = 0; k < count; k++) { G2::Pt q = pt_load<Fq2>(partials + (size_t)k * REC_BYTES + 512, 0); G2::add(acc, q); }
        G2::madd(acc, aff_load<Fq2>(consts + 5 * 64, 0));
        G2::Aff b = G2::to_affine(acc);
        store_canon(proof, 2, b.x.c0); store_canon(proof, 3, b.x.c1); store_canon(proof, 4, b.y.c0); store_canon(proof, 5, b.y.c1);
    }
}

// blockIdx.y = proof j: the scalars of its B queries (rows brows[j]) from its witness (w[1..] at wrows[j].src), through its key's
// compaction index when its B query is sparse (bidx[key] non-null), in the proof's own place of the gathered vector
__global__ void __launch_bounds__(256) gather_scalars_keyed_kernel(const fe* __restrict__ w, const KeyedRow* __restrict__ wrows, const KeyedRow* __restrict__ brows,
                                                                   const uint32_t* __restrict__ key_of, const uint32_t* const* __restrict__ bidx, fe* __restrict__ out) {
    const KeyedRow b = brows[blockIdx.y];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.n) return;
    const uint32_t* idx = bidx[key_of[blockIdx.y]];
    fe_store(&out[b.src + i], fe_load_nc(&w[wrows[blockIdx.y].src + (idx ? idx[i] : i)]));
}

// ------------------------------------------------------------------------------------------------ peer-memory exchange
constexpr size_t XCHG_SLOT = 256 + REC_BYTES;         // epoch word at +0, record at +256
constexpr size_t XCHG_BYTES = 2 * XCHG_SLOT;
// The exchange arena of a rank (one cudaMalloc, mapped by its peers through CUDA IPC):
//   [0, XCHG_BYTES)            two record slots (above)
//   XCHG_BYTES                 u32: this rank's "a peer timed out" flag (local use)
//   XCHG_BYTES + 64            u64: epoch of the evaluation vector below (release/acquire at system scope)
//   XCHG_BYTES + 256 ...       eval_cap field elements: this rank's transformed vector of the split witness map
constexpr size_t EVAL_FLAG_OFF = XCHG_BYTES + 64;
constexpr size_t EVAL_OFF = XCHG_BYTES + 256;
constexpr int MAP_RANKS = 3;                          // a, b, c are transformed on ranks 0, 1, 2

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// copy this rank's partial into its exchange slot and release the epoch (visible to peers over NVLink)
__global__ void xchg_publish_kernel(const uint8_t* __restrict__ partial, uint8_t* __restrict__ xchg, unsigned long long* __restrict__ epoch_ctr) {
    const unsigned long long epoch = *epoch_ctr + 1ull;          // every rank counts its sharded proofs the same way
    uint8_t* slot = xchg + (epoch & 1ull) * XCHG_SLOT;
    const uint4* src = reinterpret_cast<const uint4*>(partial);
    uint4* dst = reinterpret_cast<uint4*>(slot + 256);
    if (threadIdx.x < REC_BYTES / 16) dst[threadIdx.x] = src[threadIdx.x];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) { *epoch_ctr = epoch; st_release_sys(reinterpret_cast<unsigned long long*>(slot), epoch); }
}

// wait until every rank has published `epoch`, then gather the partials from peer memory (rank order) into `gathered`
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// The wait is bounded (a peer that never publishes must not wedge the GPU): after timeout_ns the rank's slot of
// `timed_out` is set and the host reports B2G_E_DEVICE.
__global__ void xchg_gather_kernel(uint8_t* const* __restrict__ peers, int count, const unsigned long long* __restrict__ epoch_ctr, uint8_t* __restrict__ gathered,
                                   unsigned long long timeout_ns, unsigned int* __restrict__ timed_out) {
    const unsigned long long epoch = *epoch_ctr;      // incremented by this rank's publish kernel just before
    const int k = blockIdx.x;                         // one CTA per rank
    const uint8_t* slot = peers[k] + (epoch & 1ull) * XCHG_SLOT;
    if (threadIdx.x == 0) {
        const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(slot);
        const unsigned long long t0 = global_timer_ns();
        while (ld_acquire_sys(flag) < epoch) {
            if (global_timer_ns() - t0 > timeout_ns) { atomicExch(timed_out, 1u + (unsigned)k); break; }
            __nanosleep(500);
        }
    }
    __syncthreads();
    if (threadIdx.x < REC_BYTES / 16) {
        const uint4* src = reinterpret_cast<const uint4*>(slot + 256);
        uint4 v;
        asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + threadIdx.x) : "memory");
        reinterpret_cast<uint4*>(gathered + (size_t)k * REC_BYTES)[threadIdx.x] = v;
    }
}

// Split witness map (sharded proofs on >= 3 GPUs).  Rank k < 3 transforms ONE of a, b, c (natural-order evaluations on H ->
// evaluations on the coset, qap.rs:60-72) into its arena and releases the epoch; every rank then forms its own slice of
// h = a*b - c (qap.rs:75-85) reading the three vectors straight out of peer HBM over NVLink: the transform work is divided by
// three, and the exchange is fused into the pointwise kernel (no collective, no host round trip).
__global__ void eval_publish_kernel(uint8_t* __restrict__ arena, const unsigned long long* __restrict__ epoch_ctr) {
    if (threadIdx.x == 0) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned long long*>(arena + EVAL_FLAG_OFF), *epoch_ctr + 1ull);
    }
}

__device__ __forceinline__ fe fe_load_sys(const void* p) {
    fe r;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]) : "l"(p) : "memory");
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]) : "l"((const char*)p + 16) : "memory");
    return r;
}

__global__ void __launch_bounds__(256) h_slice_kernel(uint8_t* const* __restrict__ peers, const unsigned long long* __restrict__ epoch_ctr, uint32_t lo, uint32_t cnt,
                                                      fe* __restrict__ h, unsigned long long timeout_ns, unsigned int* __restrict__ timed_out) {
    const unsigned long long epoch = *epoch_ctr + 1ull;
    if (threadIdx.x < MAP_RANKS) {
        const unsigned long long* flag = reinterpret_cast<const unsigned long long*>(peers[threadIdx.x] + EVAL_FLAG_OFF);
        const unsigned long long t0 = global_timer_ns();
        while (ld_acquire_sys(flag) < epoch) {
            if (global_timer_ns() - t0 > timeout_ns) { atomicExch(timed_out, 1u + threadIdx.x); break; }
            __nanosleep(200);
        }
    }
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const size_t off = EVAL_OFF + (size_t)(lo + i) * sizeof(fe);
    const fe a = fe_load_sys(peers[0] + off), b = fe_load_sys(peers[1] + off), c = fe_load_sys(peers[2] + off);
    fe_store(&h[lo + i], Fr::sub(Fr::mul(a, b), c));
}

// blockIdx.y = proof of a batch: its assignment at w + y * w_stride, its compacted scalars at out + y * n
__global__ void __launch_bounds__(256) gather_scalars_kernel(const fe* __restrict__ w, uint32_t w_stride, const uint32_t* __restrict__ idx, uint32_t n, fe* __restrict__ out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    w += (size_t)blockIdx.y * w_stride; out += (size_t)blockIdx.y * n;
    if (j < n) fe_store(&out[j], fe_load_nc(&w[idx[j]]));
}

// ------------------------------------------------------------------------------------------------ small utility kernels
template <class C, class F>
__global__ void xyzz_to_affine_kernel(const void* __restrict__ pts, uint32_t n, void* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    aff_store<F>(out, i, C::to_affine(pt_load<F>(pts, i)));
}

// out = pts[i] + pts[j] (G1 affine, 64-byte records), affine
__global__ void affine_sum_kernel(const uint8_t* __restrict__ pts, int i, int j, uint8_t* __restrict__ out) {
    G1::Pt acc = G1::from_affine(aff_load<Fq>(pts, (size_t)i));
    G1::madd(acc, aff_load<Fq>(pts, (size_t)j));
    aff_store<Fq>(out, 0, G1::to_affine(acc));
}

// Bytes per row of each test op's operands and result (0: operand not read).  XYZZ records are 4 coordinates (G1 128 B,
// G2 256 B); a G2Pair entry is a 128 B affine point followed by a 32 B word whose bit 0 is the entry's sign.
struct TestOpShape { uint32_t a, b, out, threads; };
constexpr int TEST_PAIR_RUN = 16;                          // entries one lane pair folds in op 27
constexpr uint32_t TEST_PAIR_ENTRY = 160;
static bool test_op_shape(int op, TestOpShape& s) {
    if (op < 0 || op > 29) return false;
    if (op <= 7 || (op >= 14 && op <= 16)) s = {32, (op == 6 || op == 7) ? 0u : 32u, 32, 1};
    else if (op == 8 || op == 12) s = {64, 64, 64, 1};
    else if (op == 10) s = {64, 0, 64, 1};
    else if (op == 9 || op == 13) s = {128, 128, 128, 1};
    else if (op == 11) s = {128, 0, 128, 1};
    else if (op <= 19 || op == 28) s = {64, 64, 64, 1};
    else if (op == 20) s = {128, 128, 128, 1};
    else if (op == 21) s = {128, 64, 128, 1};
    else if (op == 22) s = {128, 0, 128, 1};
    else if (op == 23) s = {256, 256, 256, 1};
    else if (op == 24) s = {256, 128, 256, 1};
    else if (op == 25) s = {256, 0, 256, 1};
    else if (op == 26) s = {256, TEST_PAIR_ENTRY, 256, 2};
    else if (op == 27) s = {TEST_PAIR_RUN * TEST_PAIR_ENTRY, 0, 256, 2};
    else s = {32, 32, 64, 1};                              // 29
    return true;
}

// the lane's coordinate of a signed G2Pair entry, negated on lane B only (as msm_accumulate_g2_kernel applies an entry's sign)
__device__ __forceinline__ fe2 test_pair_entry(const uint8_t* e, bool A) {
    fe2 qc;
    elem_load(qc, e + (A ? 0 : 64));
    const bool neg = (*reinterpret_cast<const uint32_t*>(e + 128) & 1u) != 0;
    return Fq2::sel(neg && !A, Fq2::neg(qc), qc);
}

// ops 26 / 27: lane pair `row` (threads 2 row, 2 row + 1) runs G2Pair::madd and stores the raw record as the accumulation
// kernel does (A: X, ZZ; B: Y, ZZZ)
__device__ __forceinline__ void test_op_pair(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint32_t n,
                                             uint8_t* __restrict__ out) {
    const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 1;
    if (row >= n) return;                                  // both lanes of a pair leave together
    const uint32_t half = threadIdx.x & 1u;
    const bool A = half == 0;
    const unsigned mask = 3u << (threadIdx.x & 30u);
    fe2 s0 = Fq2::zero(), s1 = Fq2::zero();
    bool empty = true;
    if (op == 26) {                                        // one addition onto a given record (empty iff ZZ == 0)
        const uint8_t* rec = a + (size_t)row * 256;
        fe2 zz; elem_load(zz, rec + 128);
        empty = Fq2::is_zero(zz);
        if (!empty) { elem_load(s0, rec + half * 64); elem_load(s1, rec + 128 + half * 64); }
        G2Pair::madd(s0, s1, empty, test_pair_entry(b + (size_t)row * TEST_PAIR_ENTRY, A), A, mask);
    } else {                                               // one run of TEST_PAIR_RUN entries from empty
        const uint8_t* run = a + (size_t)row * (TEST_PAIR_RUN * TEST_PAIR_ENTRY);
        #pragma unroll 1
        for (int k = 0; k < TEST_PAIR_RUN; k++) G2Pair::madd(s0, s1, empty, test_pair_entry(run + k * TEST_PAIR_ENTRY, A), A, mask);
    }
    uint8_t* rec = out + (size_t)row * 256;
    elem_store(rec + half * 64, s0);
    elem_store(rec + 128 + half * 64, s1);
}

__global__ void test_op_kernel(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint32_t n, uint8_t* __restrict__ out) {
    if (op == 26 || op == 27) { test_op_pair(op, a, b, n, out); return; }
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (op <= 7) {
        fe x = fe_load(a + 32 * (size_t)i), y = (op == 6 || op == 7) ? fe_zero() : fe_load(b + 32 * (size_t)i), r;
        switch (op) {
            case 0: r = Fq::mul(x, y); break;
            case 1: r = Fq::add(x, y); break;
            case 2: r = Fq::sub(x, y); break;
            case 3: r = Fr::mul(x, y); break;
            case 4: r = Fr::add(x, y); break;
            case 5: r = Fr::sub(x, y); break;
            case 6: r = Fq::inv(x); break;
            default: r = Fr::inv(x); break;
        }
        fe_store(out + 32 * (size_t)i, r);
    } else if (op == 8 || op == 10) {
        G1::Aff p = aff_load<Fq>(a, i);
        G1::Pt acc = G1::from_affine(p);
        if (op == 8) { G1::Pt q = G1::from_affine(aff_load<Fq>(b, i)); G1::add(acc, q); }   // exercises the full addition
        else acc = G1::dbl(acc);
        aff_store<Fq>(out, i, G1::to_affine(acc));
    } else if (op == 9 || op == 11) {
        G2::Aff p = aff_load<Fq2>(a, i);
        G2::Pt acc = G2::from_affine(p);
        if (op == 9) { G2::Pt q = G2::from_affine(aff_load<Fq2>(b, i)); G2::add(acc, q); }
        else acc = G2::dbl(acc);
        aff_store<Fq2>(out, i, G2::to_affine(acc));
    } else if (op == 12) {      // mixed addition path
        G1::Pt acc = G1::from_affine(aff_load<Fq>(a, i));
        G1::madd(acc, aff_load<Fq>(b, i));
        aff_store<Fq>(out, i, G1::to_affine(acc));
    } else if (op == 13) {
        G2::Pt acc = G2::from_affine(aff_load<Fq2>(a, i));
        G2::madd(acc, aff_load<Fq2>(b, i));
        aff_store<Fq2>(out, i, G2::to_affine(acc));
    } else if (op <= 16) {      // the lazy-reduction blocks on raw Montgomery residues
        fe x = fe_load(a + 32 * (size_t)i), y = fe_load(b + 32 * (size_t)i), r;
        if (op == 14) r = Fq::sqr(x);
        else if (op == 15) r = Fq::mul_sub(x, y, y, y);
        else { uint32_t t[16]; Fq::mul_wide(t, x, y); r = Fq::redc(t); }
        fe_store(out + 32 * (size_t)i, r);
    } else if (op <= 19 || op == 28) {   // 17 fq2_mul, 18 fq2_sqr, 19 fq2_mul_sub(a, b, b, swap(a)), 28 fq2_mul_inline
        fe2 x, y, r;
        x.c0 = fe_load(a + 64 * (size_t)i); x.c1 = fe_load(a + 64 * (size_t)i + 32);
        y.c0 = fe_load(b + 64 * (size_t)i); y.c1 = fe_load(b + 64 * (size_t)i + 32);
        if (op == 17) r = Fq2::mul(x, y);
        else if (op == 18) r = Fq2::sqr(x);
        else if (op == 28) r = Fq2::mul_inline(x, y);
        else { fe2 z; z.c0 = x.c1; z.c1 = x.c0; r = Fq2::mul_sub(x, y, y, z); }
        fe_store(out + 64 * (size_t)i, r.c0); fe_store(out + 64 * (size_t)i + 32, r.c1);
    } else if (op <= 22) {      // G1 on raw XYZZ records, result not normalised: 20 add(a, b), 21 madd(a, affine b), 22 dbl(a)
        G1::Pt acc = pt_load<Fq>(a, i);
        if (op == 20) { G1::Pt q = pt_load<Fq>(b, i); G1::add(acc, q); }
        else if (op == 21) G1::madd(acc, aff_load<Fq>(b, i));
        else acc = G1::dbl(acc);
        pt_store<Fq>(out, i, acc);
    } else if (op <= 25) {      // the same for G2: 23 add, 24 madd, 25 dbl
        G2::Pt acc = pt_load<Fq2>(a, i);
        if (op == 23) { G2::Pt q = pt_load<Fq2>(b, i); G2::add(acc, q); }
        else if (op == 24) G2::madd(acc, aff_load<Fq2>(b, i));
        else acc = G2::dbl(acc);
        pt_store<Fq2>(out, i, acc);
    } else {                    // 29: the plain 512-bit product a * b (a < 2^255)
        uint32_t t[16];
        Fq::mul_wide(t, fe_load(a + 32 * (size_t)i), fe_load(b + 32 * (size_t)i));
        fe lo, hi;
        #pragma unroll
        for (int k = 0; k < 8; k++) { lo.l[k] = t[k]; hi.l[k] = t[8 + k]; }
        fe_store(out + 64 * (size_t)i, lo); fe_store(out + 64 * (size_t)i + 32, hi);
    }
}

// ------------------------------------------------------------------------------------------------ host helpers
// witness and witness-map vectors of `count` proofs (assignments n_vars apart, a / b / c / h n apart)
static void ensure_witness_buffers(b2g_ctx* ctx, size_t n_vars, size_t n, uint32_t count = 1) {
    n_vars *= count; n *= count;
    if (n_vars > ctx->cap_w) {
        if (ctx->d_w) cudaFree(ctx->d_w);
        ctx->d_w = nullptr; ctx->cap_w = 0;
        CUDA_CHECK(cudaMalloc(&ctx->d_w, (n_vars + 1) * sizeof(fe)));
        ctx->cap_w = n_vars; ctx->alloc_gen++;
    }
    if (n > ctx->cap_n) {
        ctx->cap_n = 0;
        for (fe** p : {&ctx->d_a, &ctx->d_b, &ctx->d_c, &ctx->d_h}) if (*p) { cudaFree(*p); *p = nullptr; }
        for (fe** p : {&ctx->d_a, &ctx->d_b, &ctx->d_c, &ctx->d_h}) CUDA_CHECK(cudaMalloc(p, n * sizeof(fe)));
        ctx->cap_n = n; ctx->alloc_gen++;
    }
}

// the per-proof records, proof slots, (r, s) and glue precomputation of `count` proofs; grown on demand, never shrunk
static void ensure_batch_buffers(b2g_ctx* ctx, uint32_t count) {
    if (count <= ctx->cap_batch) return;
    CUDA_CHECK(cudaDeviceSynchronize());
    for (uint8_t** p : {&ctx->d_partial, &ctx->d_proof, &ctx->d_pre, &ctx->d_rs}) { cudaFree(*p); *p = nullptr; }
    for (uint8_t** p : {&ctx->h_rs, &ctx->h_proof}) { cudaFreeHost(*p); *p = nullptr; }
    ctx->cap_batch = 0; ctx->alloc_gen++;
    if (ctx->scratch_ok) for (int q = 0; q < NQ; q++) ctx->scratch[q].result = nullptr;
    CUDA_CHECK(cudaMalloc(&ctx->d_partial, count * REC_BYTES));
    CUDA_CHECK(cudaMemset(ctx->d_partial, 0, count * REC_BYTES));
    CUDA_CHECK(cudaMalloc(&ctx->d_proof, count * 256));
    CUDA_CHECK(cudaMalloc(&ctx->d_pre, count * PRE_BYTES));
    CUDA_CHECK(cudaMalloc(&ctx->d_rs, count * 64));
    CUDA_CHECK(cudaMallocHost(&ctx->h_rs, count * 64));
    CUDA_CHECK(cudaMallocHost(&ctx->h_proof, count * 256));
    ctx->cap_batch = count;
    if (ctx->scratch_ok) for (int q = 0; q < NQ; q++) ctx->scratch[q].result = ctx->d_partial + PARTIAL_OFF[q];
}

// per-stream MSM scratch of this context for `count` proofs: query q at plan[q]'s window size and buckets with n[q] bases per
// proof; H and L with sort buffers, and B1 too when bsort (B1 and B2 then read a B sort of their own, over nwb gathered B
// scalars in d_wb; otherwise they read L's).  Kept while later calls fit (a smaller batch reuses it); re-created for exactly
// this call when they do not, so a larger key after a large batch does not inherit that batch's size.
static void ensure_scratch(b2g_ctx* ctx, const MsmPlan* plan, const uint32_t* n, uint32_t count, bool bsort, size_t nwb) {
    bool ok = ctx->scratch_ok && (!bsort || (ctx->scratch_bsort && nwb <= ctx->cap_wb));
    for (int q = 0; q < NQ && ok; q++) {
        const MsmPlan& p = plan[q]; const MsmScratch& sc = ctx->scratch[q];
        if (n[q] > sc.cap_n || p.nwin > sc.cap_nwin || p.nbuckets > sc.cap_buckets || count > sc.cap_count) ok = false;
    }
    if (ok) return;
    CUDA_CHECK(cudaDeviceSynchronize());
    for (int q = 0; q < NQ; q++) msm_scratch_free(ctx->scratch[q]);     // also the remains of an allocation that failed
    ctx->scratch_ok = false; ctx->alloc_gen++;
    for (int q = 0; q < NQ; q++) {
        msm_scratch_alloc(ctx->scratch[q], n[q], plan[q].nwin, plan[q].nbuckets, q == Q_B2, q == Q_H || q == Q_L || (q == Q_B1 && bsort), count);
        cudaFree(ctx->scratch[q].result);
        ctx->scratch[q].result = ctx->d_partial + PARTIAL_OFF[q];
        ctx->scratch[q].result_owned = false;
        ctx->scratch[q].result_stride = REC_BYTES;
    }
    ctx->scratch_bsort = bsort;
    if (nwb > ctx->cap_wb) {
        if (ctx->d_wb) cudaFree(ctx->d_wb);
        ctx->d_wb = nullptr; ctx->cap_wb = 0;
        CUDA_CHECK(cudaMalloc(&ctx->d_wb, (nwb + 1) * sizeof(fe)));
        ctx->cap_wb = nwb;
    }
    ctx->scratch_ok = true;
}

// the scratch of `count` proofs under one key
static void ensure_scratch(b2g_ctx* ctx, const b2g_pk* pk, uint32_t count = 1) {
    uint32_t n[NQ];
    for (int q = 0; q < NQ; q++) n[q] = pk->plan[q].n ? pk->plan[q].n : 1;
    ensure_scratch(ctx, pk->plan, n, count, pk->d_bidx != nullptr, (size_t)pk->b_compact * count);
}

// the witness map of `count` proofs side by side: one launch per kernel of the chain, the batch on a grid dimension.  The
// first witness at d_w + w_off, the first a / b / c / h vector at v_off (b2g_prove_keys: one key's proofs of a keyed batch).
static void run_witness_map(b2g_ctx* ctx, b2g_mat* mat, cudaStream_t st, uint32_t count = 1, size_t w_off = 0, size_t v_off = 0) {
    fe *w = ctx->d_w + w_off, *a = ctx->d_a + v_off, *b = ctx->d_b + v_off, *c = ctx->d_c + v_off, *h = ctx->d_h + v_off;
    if (mat->reduction == B2G_REDUCTION_LIBSNARK) {
        spmv_launch(mat->n, mat->m, mat->num_inputs, mat->a_rowptr, mat->a_col, mat->a_val, mat->b_rowptr, mat->b_col, mat->b_val,
                    w, a, b, c, st, mat->c_rowptr, mat->c_col, mat->c_val, count, mat->n_vars);
        ntt_witness_transform_libsnark(mat->dom, a, b, c, a, h, st, count);   // a doubles as scratch
        return;
    }
    spmv_launch(mat->n, mat->m, mat->num_inputs, mat->a_rowptr, mat->a_col, mat->a_val, mat->b_rowptr, mat->b_col, mat->b_val,
                w, a, b, c, st, nullptr, nullptr, nullptr, count, mat->n_vars);
    ntt_witness_transform(mat->dom, a, b, c, h, st, count);
}

// a key's tables live on one device and describe one shard: checked before the first kernel that dereferences them
static void check_pk_ctx(const b2g_ctx* ctx, const b2g_pk* pk) {
    if (!ctx || !pk) throw_error(B2G_E_SHAPE, "null handle");
    if (pk->device != ctx->device) throw_error(B2G_E_SHAPE, "handle belongs to another device");
    if (pk->shard_rank != ctx->shard_rank || pk->shard_count != ctx->shard_count) throw_error(B2G_E_SHAPE, "proving key was loaded for another shard");
}

static void check_shapes(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat) {
    if (!ctx || !pk || !mat) throw_error(B2G_E_SHAPE, "null handle");
    check_pk_ctx(ctx, pk);
    if (mat->device != ctx->device) throw_error(B2G_E_SHAPE, "handle belongs to another device");
    if (pk->n_vars != mat->n_vars) throw_error(B2G_E_SHAPE, "proving key and matrices disagree on n_vars");
    if (mat->reduction == B2G_REDUCTION_LIBSNARK) {
        // arkworks keys carry domain - 1 H bases; msm_bigint pairs min(len) terms (the top coefficient of h is zero)
        if (pk->domain + 1 != mat->n && pk->domain != mat->n) throw_error(B2G_E_SHAPE, "H query length must be domain_size - 1 (or domain_size) for LibsnarkReduction");
    } else if (pk->domain != mat->n) throw_error(B2G_E_SHAPE, "proving key domain_size != next_pow2(num_constraints + num_inputs)");
    if (pk->n_public + 1 != mat->num_inputs) throw_error(B2G_E_SHAPE, "proving key n_public + 1 != num_inputs");
}

// device part of a proof up to the five partial MSM results (witness must already be in ctx->d_w).
// The four witness-scalar queries (L, A, B1, B2) are defined over the same index range and share ONE digit sort.
// Launch order of the four witness MSMs.  Each is a GPU-filling accumulation followed by a latency chain on a few CTAs (fold,
// bucket reduction, and for A / B1 the scalar multiplication by s / r; B2's tail is shorter, L's the shortest).  The chains with
// the longest tails go first so that their tails run under the accumulations that follow: A, B1, B2, L.  On one GPU at 2^20 the
// accumulations are long enough to hide every tail; in one shard of a many-way sharded proof they are short and the order
// decides which tail sticks out.
static const int WITNESS_ORDER[4] = {Q_A, Q_B1, Q_B2, Q_L};

// scale: also compute s*msm_A and r*msm_B1 (d_rs must hold r, s) on those MSMs' own streams, right behind them
static unsigned long long p2p_timeout_ns() {
    const char* v = getenv("B2G_P2P_TIMEOUT_MS");
    long ms = v && *v ? strtol(v, nullptr, 10) : 20000;
    return (unsigned long long)(ms > 0 ? ms : 20000) * 1000000ull;
}

static bool map_is_split(const b2g_ctx* ctx, const b2g_mat* mat) {
    return ctx->shard_count >= MAP_RANKS && ctx->peers_imported == ctx->shard_count && mat->reduction == B2G_REDUCTION_CIRCOM &&
           ctx->eval_common >= mat->n;
}

// witness map of a sharded proof with the three transforms on ranks 0, 1, 2 (kernels above); fills d_h[lo, lo + cnt) only
static void run_witness_map_split(b2g_ctx* ctx, b2g_mat* mat, uint32_t lo, uint32_t cnt, cudaStream_t st) {
    const int rank = ctx->shard_rank;
    unsigned int* d_flag = reinterpret_cast<unsigned int*>(ctx->d_xchg + XCHG_BYTES);
    if (rank < MAP_RANKS) {
        fe* eval = reinterpret_cast<fe*>(ctx->d_xchg + EVAL_OFF);
        spmv_launch(mat->n, mat->m, mat->num_inputs, mat->a_rowptr, mat->a_col, mat->a_val, mat->b_rowptr, mat->b_col, mat->b_val, ctx->d_w,
                    rank == 0 ? eval : ctx->d_a, rank == 1 ? eval : ctx->d_b, rank == 2 ? eval : ctx->d_c, st);
        ntt_transform_single(mat->dom, eval, st);
        eval_publish_kernel<<<1, 32, 0, st>>>(ctx->d_xchg, ctx->d_epoch);
        g_launch_count += 1;
    }
    if (cnt) {
        h_slice_kernel<<<(cnt + 255) / 256, 256, 0, st>>>(ctx->d_peer_ptrs, ctx->d_epoch, lo, cnt, ctx->d_h, p2p_timeout_ns(), d_flag);
        g_launch_count += 1;
    }
    CUDA_CHECK(cudaGetLastError());
}

// The four witness-query accumulations of `count` proofs in WITNESS_ORDER, each on its own stream behind the sort it reads:
// the W sort (ev_sort, on the L stream) or, when bsort, for B1 and B2 the B sort (ev_sortb, on the B1 stream).  Each ends in
// ev_done[q].  scale: s*msm_A and r*msm_B1 right behind those MSMs (d_rs must hold r, s); timed: phase events around each.
static void accumulate_witness_queries(b2g_ctx* ctx, const MsmPlan* plan, bool bsort, uint32_t count, bool timed, bool scale) {
    for (int q : WITNESS_ORDER) {
        const bool on_b = bsort && (q == Q_B1 || q == Q_B2);
        if (on_b) { if (q != Q_B1) CUDA_CHECK(cudaStreamWaitEvent(ctx->st[q], ctx->ev_sortb, 0)); }
        else if (q != Q_L) CUDA_CHECK(cudaStreamWaitEvent(ctx->st[q], ctx->ev_sort, 0));
        if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[2 * q], ctx->st[q]));
        msm_accumulate(plan[q], on_b ? ctx->scratch[Q_B1] : ctx->scratch[Q_L], ctx->scratch[q], ctx->st[q]);
        if (scale && (q == Q_A || q == Q_B1)) {
            const Scalar256* rs = reinterpret_cast<const Scalar256*>(ctx->d_rs);
            scale_partial_kernel<<<count, 32, 0, ctx->st[q]>>>(ctx->d_partial + PARTIAL_OFF[q], q == Q_A ? rs + 1 : rs, ctx->d_partial + B2G_PARTIAL_BYTES + (q == Q_A ? 0 : 128), 2);
            g_launch_count += 1;
        }
        if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[2 * q + 1], ctx->st[q]));
        CUDA_CHECK(cudaEventRecord(ctx->ev_done[q], ctx->st[q]));
    }
}

// count > 1: a batch of proofs (witnesses pk->n_vars apart in d_w); every MSM sorts and accumulates the whole batch at once
static void launch_msms(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, bool timed, bool scale, bool split_map = false, uint32_t count = 1) {
    cudaStream_t s0 = ctx->st[0], ssort = ctx->st[Q_L];
    CUDA_CHECK(cudaEventRecord(ctx->ev_w, s0));
    CUDA_CHECK(cudaStreamWaitEvent(ssort, ctx->ev_w, 0));
    msm_sort(pk->plan[Q_A], ctx->scratch[Q_L], ctx->d_w + pk->scalar_off[Q_A] + pk->lo[Q_A], pk->cnt[Q_A], true, ssort, count, pk->n_vars);
    CUDA_CHECK(cudaEventRecord(ctx->ev_sort, ssort));
    const bool bsparse = pk->d_bidx != nullptr;
    if (bsparse) {
        // B1 and B2 over the compacted base set: gather their scalars and sort them separately (on the B1 stream)
        cudaStream_t sb = ctx->st[Q_B1];
        CUDA_CHECK(cudaStreamWaitEvent(sb, ctx->ev_w, 0));
        if (pk->b_compact) gather_scalars_kernel<<<dim3((pk->b_compact + 255) / 256, count), 256, 0, sb>>>(ctx->d_w + pk->scalar_off[Q_B1] + pk->lo[Q_B1], pk->n_vars, pk->d_bidx, pk->b_compact, ctx->d_wb);
        g_launch_count += 1;
        msm_sort(pk->plan[Q_B1], ctx->scratch[Q_B1], ctx->d_wb, pk->b_compact, true, sb, count, pk->b_compact);
        CUDA_CHECK(cudaEventRecord(ctx->ev_sortb, sb));
    }
    accumulate_witness_queries(ctx, pk->plan, bsparse, count, timed, scale);
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[10], s0));
    if (split_map) run_witness_map_split(ctx, mat, pk->lo[Q_H], pk->cnt[Q_H], s0);
    else run_witness_map(ctx, mat, s0, count);
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[11], s0));
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[0], s0));
    msm_run(pk->plan[Q_H], ctx->scratch[Q_H], ctx->d_h + pk->lo[Q_H], pk->cnt[Q_H], true, s0, count, mat->n);   // pairs min(#bases, #h) terms
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[1], s0));
    for (int q = 1; q < NQ; q++) CUDA_CHECK(cudaStreamWaitEvent(s0, ctx->ev_done[q], 0));
}

// frees every device allocation of a (possibly partially built) key and the key itself
static void pk_release(b2g_pk* pk) {
    for (int q = 0; q < NQ; q++) msm_free_table(pk->plan[q]);
    if (pk->d_consts) cudaFree(pk->d_consts);
    if (pk->d_tab_delta1) cudaFree(pk->d_tab_delta1);
    if (pk->d_tab_delta2) cudaFree(pk->d_tab_delta2);
    if (pk->d_tab_aa) cudaFree(pk->d_tab_aa);
    if (pk->d_tab_bb) cudaFree(pk->d_tab_bb);
    if (pk->d_bidx) cudaFree(pk->d_bidx);
    delete pk;
}


// Sparse B: the support of the B polynomials inside a shard's range [lo, lo + cnt) of w[1..] (a base counts if it is a real
// point in either group).  True when fewer than 80 % of them are real: then idx = their positions and packed = their G1 / G2
// bases side by side.
static bool b_support(const b2g_pk_desc* d, uint32_t lo, uint32_t cnt, std::vector<uint32_t>& idx, std::vector<uint8_t> packed[2]) {
    const uint8_t* b1 = (const uint8_t*)d->b_g1_query + (size_t)(1 + lo) * 64;
    const uint8_t* b2 = (const uint8_t*)d->b_g2_query + (size_t)(1 + lo) * 128;
    auto nonzero = [](const uint8_t* p, size_t n) { const uint64_t* w = (const uint64_t*)p; uint64_t o = 0; for (size_t i = 0; i < n / 8; i++) o |= w[i]; return o != 0; };
    idx.clear();
    for (uint32_t i = 0; i < cnt; i++) if (nonzero(b1 + (size_t)i * 64, 64) || nonzero(b2 + (size_t)i * 128, 128)) idx.push_back(i);
    const char* off = getenv("B2G_NO_B_COMPACT");
    if (!(off && *off == '1') && cnt >= 1024 && (uint64_t)idx.size() * 5 < (uint64_t)cnt * 4) {
        packed[0].resize(idx.size() * 64 + 64); packed[1].resize(idx.size() * 128 + 128);
        for (size_t j = 0; j < idx.size(); j++) { memcpy(&packed[0][j * 64], b1 + (size_t)idx[j] * 64, 64); memcpy(&packed[1][j * 128], b2 + (size_t)idx[j] * 128, 128); }
        return true;
    }
    idx.clear();
    return false;
}

// a key's glue constants and the 8-bit window tables of its fixed bases (delta_g1, delta_g2, alpha_g1 + a_query[0],
// beta_g1 + b_g1_query[0]); synchronises `st`
static void pk_load_glue(b2g_pk* pk, const b2g_pk_desc* d, cudaStream_t st) {
    std::vector<uint8_t> consts(5 * 64 + 3 * 128);
    memcpy(&consts[0], d->alpha_g1, 64); memcpy(&consts[64], d->beta_g1, 64); memcpy(&consts[128], d->delta_g1, 64);
    memcpy(&consts[192], d->a_query, 64); memcpy(&consts[256], d->b_g1_query, 64);
    memcpy(&consts[320], d->beta_g2, 128); memcpy(&consts[448], d->delta_g2, 128); memcpy(&consts[576], d->b_g2_query, 128);
    pk->d_consts = dev_upload<uint8_t>(consts.data(), consts.size(), st);
    // alpha, beta, delta and the three query[0] points never pass through a table build: G1Affine::new / G2Affine::new
    // validate them in the reference (src/zkey.rs:340-360), so they are checked here as well
    msm_validate_points(pk->d_consts, 5, false, st, "alpha_g1 / beta_g1 / delta_g1 / a_query[0] / b_g1_query[0]");
    msm_validate_points(pk->d_consts + 5 * 64, 3, true, st, "beta_g2 / delta_g2 / b_g2_query[0]");
    CUDA_CHECK(cudaMalloc(&pk->d_tab_delta1, 32 * 255 * 64));
    CUDA_CHECK(cudaMalloc(&pk->d_tab_delta2, 32 * 255 * 128));
    CUDA_CHECK(cudaMalloc(&pk->d_tab_aa, 32 * 255 * 64 + 64));
    CUDA_CHECK(cudaMalloc(&pk->d_tab_bb, 32 * 255 * 64 + 64));
    fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(pk->d_tab_delta1, pk->d_consts + 2 * 64);
    fixed_table_kernel<G2, Fq2><<<(32 * 255 + 63) / 64, 64, 0, st>>>(pk->d_tab_delta2, pk->d_consts + 5 * 64 + 128);
    // alpha1 + a_query[0] and beta1 + b_g1_query[0] (affine sums parked behind their tables), then their window tables
    affine_sum_kernel<<<1, 1, 0, st>>>(pk->d_consts, 0, 3, (uint8_t*)pk->d_tab_aa + 32 * 255 * 64);
    affine_sum_kernel<<<1, 1, 0, st>>>(pk->d_consts, 1, 4, (uint8_t*)pk->d_tab_bb + 32 * 255 * 64);
    fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(pk->d_tab_aa, (uint8_t*)pk->d_tab_aa + 32 * 255 * 64);
    fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(pk->d_tab_bb, (uint8_t*)pk->d_tab_bb + 32 * 255 * 64);
    g_launch_count += 6;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// header checks of a proving-key descriptor (b2g_pk_load, b2g_pk_group_load)
static void pk_desc_check(const b2g_pk_desc* d) {
    if (d->n_vars < d->n_public + 1 || d->domain_size == 0) throw_error(B2G_E_SHAPE, "bad proving-key header");
    for (const void* p : {d->alpha_g1, d->beta_g1, d->delta_g1, d->beta_g2, d->delta_g2, d->a_query, d->b_g1_query, d->b_g2_query, d->h_query})
        if (!p) throw_error(B2G_E_SHAPE, "null proving-key section");
    if (d->n_vars - (d->n_public + 1) && !d->l_query) throw_error(B2G_E_SHAPE, "null proving-key section");
}

// L, A, B1, B2 all pair bases with w[1..n_vars): L is re-indexed onto that range by prepending (l - 1) points at infinity
// (l_query[j] belongs to w[l + j]), so the four queries share one digit sort per proof
static std::vector<uint8_t> l_padded(const b2g_pk_desc* d) {
    const uint32_t li = d->n_public + 1;
    std::vector<uint8_t> l((size_t)(d->n_vars - 1) * 64, 0);
    if (d->n_vars - li) memcpy(l.data() + (size_t)(li - 1) * 64, d->l_query, (size_t)(d->n_vars - li) * 64);
    return l;
}

// one query's table from n host bases of `aff` bytes: uploaded to tmp (which a caller's guard frees if a step throws),
// build(tmp), synchronise, free tmp
template <class Build>
static void table_from_host(void*& tmp, const void* src, uint32_t n, size_t aff, cudaStream_t st, Build build) {
    if (n) tmp = dev_upload<uint8_t>(src, (size_t)n * aff, st);
    build(tmp);
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (tmp) { cudaFree(tmp); tmp = nullptr; }
}

// (r, s) -> ctx->d_rs on stream 0.  Every entry point synchronises stream 0 before it returns (b2g_bench_device stages once),
// so the pinned staging slot is free again by the time the next call overwrites it.  count proofs: r, s = count x 32 B each,
// staged as r_j | s_j pairs.
static void stage_rs(b2g_ctx* ctx, const void* r, const void* s, uint32_t count = 1) {
    for (uint32_t j = 0; j < count; j++) {
        memcpy(ctx->h_rs + 64 * j, (const uint8_t*)r + 32 * j, 32);
        memcpy(ctx->h_rs + 64 * j + 32, (const uint8_t*)s + 32 * j, 32);
    }
    CUDA_CHECK(cudaMemcpyAsync(ctx->d_rs, ctx->h_rs, 64 * (size_t)count, cudaMemcpyHostToDevice, ctx->st[0]));
    memcpy(ctx->pre_r, r, 32); memcpy(ctx->pre_s, s, 32);
}

// r*delta1, K_C and s*delta2 depend only on (r, s): launch(st_glue) enqueues the glue_pre kernel on a side stream forked from
// stream 0 (after d_rs is written and after the previous proof's assembly has read d_pre), so it overlaps the MSMs; ev_pre
// marks its end
template <class Launch>
static void fork_glue_pre(b2g_ctx* ctx, Launch launch) {
    CUDA_CHECK(cudaEventRecord(ctx->ev_fork, ctx->st[0]));
    CUDA_CHECK(cudaStreamWaitEvent(ctx->st_glue, ctx->ev_fork, 0));
    launch(ctx->st_glue);
    CUDA_CHECK(cudaEventRecord(ctx->ev_pre, ctx->st_glue));
    g_launch_count += 1;
}

// launch() enqueues the glue_post kernel on `st` once glue_pre is in
template <class Launch>
static void join_glue_post(b2g_ctx* ctx, cudaStream_t st, Launch launch) {
    CUDA_CHECK(cudaStreamWaitEvent(st, ctx->ev_pre, 0));
    launch();
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

static void launch_glue_pre(b2g_ctx* ctx, b2g_pk* pk, uint32_t count = 1) {
    fork_glue_pre(ctx, [&](cudaStream_t sg) {
        glue_pre_kernel<<<count, 160, 0, sg>>>(pk->d_tab_delta1, pk->d_tab_delta2, pk->d_tab_aa, pk->d_tab_bb, reinterpret_cast<const Scalar256*>(ctx->d_rs), ctx->d_pre);
    });
    ctx->pre_valid = true;
}

// partials_dev: `count` records of REC_BYTES per proof; nproofs > 1: proofs of a batch, each assembled from its own records
static void launch_glue_post(b2g_ctx* ctx, b2g_pk* pk, const uint8_t* partials_dev, int count, cudaStream_t st, uint32_t nproofs = 1) {
    join_glue_post(ctx, st, [&] { glue_post_kernel<<<nproofs, 96, 0, st>>>(partials_dev, count, pk->d_consts, ctx->d_pre, ctx->d_proof); });
}

// Everything one proof does on the device between "witness and (r, s) are in HBM" and "proof bytes are in d_proof".
// kind 0: whole proof, or `count` whole proofs of a batch; kind 1: base-sharded proof whose partials are exchanged through
// NVLink peer memory.
static void enqueue_proof(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int kind, bool timed, uint32_t count = 1) {
    cudaStream_t s0 = ctx->st[0];
    unsigned int* d_flag = kind == 1 ? reinterpret_cast<unsigned int*>(ctx->d_xchg + XCHG_BYTES) : nullptr;   // local word after the two slots
    if (kind == 1) CUDA_CHECK(cudaMemsetAsync(d_flag, 0, 4, s0));
    launch_glue_pre(ctx, pk, count);
    launch_msms(ctx, pk, mat, timed, true, kind == 1 && map_is_split(ctx, mat), count);
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[14], s0));
    if (kind == 1) {
        xchg_publish_kernel<<<1, 64, 0, s0>>>(ctx->d_partial, ctx->d_xchg, ctx->d_epoch);
        xchg_gather_kernel<<<ctx->shard_count, 64, 0, s0>>>(ctx->d_peer_ptrs, ctx->shard_count, ctx->d_epoch, ctx->d_partials_all, p2p_timeout_ns(), d_flag);
        g_launch_count += 2;
        launch_glue_post(ctx, pk, ctx->d_partials_all, ctx->shard_count, s0);
    } else {
        launch_glue_post(ctx, pk, ctx->d_partial, 1, s0, count);
    }
}

// Replays the pass captured in `slot` (capturing enqueue(false) first if the slot holds none for `key`); runs enqueue(true)
// directly when graphs are disabled or the capture fails.  timers: the pass has phase timers, recorded around the replay.
template <class Enqueue>
static void run_graph(b2g_ctx* ctx, GraphSlot& slot, std::vector<uint64_t> key, bool timers, Enqueue enqueue) {
    cudaStream_t s0 = ctx->st[0];
    if (!ctx->use_graph) { enqueue(true); return; }
    if (slot.exec && slot.key != key) { cudaGraphExecDestroy(slot.exec); slot.exec = nullptr; }
    if (!slot.exec) {
        const uint64_t before = g_launch_count.load();
        cudaGraph_t graph = nullptr;
        CUDA_CHECK(cudaStreamBeginCapture(s0, cudaStreamCaptureModeThreadLocal));
        try { enqueue(false); }
        catch (...) { cudaStreamEndCapture(s0, &graph); if (graph) cudaGraphDestroy(graph); cudaGetLastError(); g_launch_count = before; throw; }
        cudaError_t e = cudaStreamEndCapture(s0, &graph);
        if (e == cudaSuccess) e = cudaGraphInstantiate(&slot.exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        slot.launches = g_launch_count.load() - before;
        g_launch_count = before;
        if (e != cudaSuccess) {                       // not fatal: run this context without graphs from now on
            cudaGetLastError();
            slot.exec = nullptr; ctx->use_graph = false;
            enqueue(true);
            return;
        }
        slot.key = std::move(key);
    }
    if (timers) {
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[10], s0)); CUDA_CHECK(cudaEventRecord(ctx->ev_t[11], s0));    // phase timers are not part of the graph:
        for (int i = 0; i < 10; i++) CUDA_CHECK(cudaEventRecord(ctx->ev_t[i], s0));                         // they read as zero
    }
    CUDA_CHECK(cudaGraphLaunch(slot.exec, s0));
    if (timers) CUDA_CHECK(cudaEventRecord(ctx->ev_t[14], s0));
    g_launch_count += slot.launches;
}

// kind 0 (G_PROOF) or 1 (G_P2P), as enqueue_proof takes it
static void run_proof(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int kind, uint32_t count = 1) {
    run_graph(ctx, ctx->graphs[kind], {pk->uid, mat->uid, ctx->alloc_gen, count}, true,
              [&](bool timed) { enqueue_proof(ctx, pk, mat, kind, timed, count); });
}

static void collect_timings(b2g_ctx* ctx) {
    auto el = [&](int a, int b) { float ms = 0; cudaEventElapsedTime(&ms, ctx->ev_t[a], ctx->ev_t[b]); return ms; };
    ctx->last_ms[0] = el(12, 13);           // h2d
    ctx->last_ms[1] = el(10, 11);           // witness map
    ctx->last_ms[2] = el(0, 1);             // msm H
    for (int q = 1; q < NQ; q++) ctx->last_ms[2 + q] = el(2 * q, 2 * q + 1);
    ctx->last_ms[7] = el(14, 15);           // glue + d2h
    ctx->last_ms[8] = el(12, 15);           // whole call
}

// The body of b2g_prove_many and b2g_prove_keys once their arguments are checked: grow() sizes the buffers (an out-of-memory
// error is reworded to name the call's proofs, and for b2g_prove_keys its n_keys keys), the witnesses are
// uploaded back to back (witness j: n_vars[key_of[j]] elements, key_of null for one key), (r, s) are staged, run() enqueues
// the pass, and the count x 256 proof bytes are copied to the pinned slot h_proof.  Nothing here waits for the device.
// timed: phase timers around the upload.
template <class Grow, class Run>
static void prove_pass(b2g_ctx* ctx, uint32_t count, size_t n_keys, bool timed, const void* r_canon, const void* s_canon, const void* const* w_mont,
                       const uint32_t* n_vars, const uint32_t* key_of, Grow grow, Run run) {
    try {
        grow();
    } catch (const B2gError& e) {
        if (e.code != B2G_E_DEVICE) throw;
        cudaGetLastError();
        throw_error(B2G_E_DEVICE, "the device buffers of " + std::to_string(count) + " proof(s)" +
                                  (n_keys ? " under " + std::to_string(n_keys) + " key(s)" : std::string()) + " do not fit in device memory" +
                                  (count > 1 || n_keys ? "; prove fewer per call (" : " (") + e.what() + ")");
    }
    cudaStream_t s0 = ctx->st[0];
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[12], s0));
    size_t at = 0;
    for (uint32_t j = 0; j < count; j++) {
        const size_t n = n_vars[key_of ? key_of[j] : 0];
        CUDA_CHECK(cudaMemcpyAsync(ctx->d_w + at, w_mont[j], n * 32, cudaMemcpyHostToDevice, s0));
        at += n;
    }
    if (timed) CUDA_CHECK(cudaEventRecord(ctx->ev_t[13], s0));
    stage_rs(ctx, r_canon, s_canon, count);
    run();
    ctx->pre_valid = false;
    CUDA_CHECK(cudaMemcpyAsync(ctx->h_proof, ctx->d_proof, (size_t)count * 256, cudaMemcpyDeviceToHost, s0));
}

}  // namespace b2g

// ================================================================================================== C ABI
extern "C" {

const char* b2g_last_error(void) { return g_last_error.c_str(); }
int b2g_version(void) { return 1; }

int b2g_device_count(int* count) {
    return guarded([&] { if (!count) throw_error(B2G_E_SHAPE, "null pointer"); CUDA_CHECK(cudaGetDeviceCount(count)); });
}

int b2g_ctx_create(int device, int shard_rank, int shard_count, b2g_ctx** out) {
    return guarded([&] {
        if (!out) throw_error(B2G_E_SHAPE, "null pointer");
        if (shard_count < 1 || shard_count > 64 || shard_rank < 0 || shard_rank >= shard_count) throw_error(B2G_E_SHAPE, "bad shard rank/count");
        int ndev = 0;
        CUDA_CHECK(cudaGetDeviceCount(&ndev));
        if (device < 0 || device >= ndev) throw_error(B2G_E_DEVICE, "no such CUDA device (this library has no CPU fallback)");
        DevGuard g(device);
        b2g_ctx* ctx = new b2g_ctx();
        ctx->device = device; ctx->shard_rank = shard_rank; ctx->shard_count = shard_count;
        // the proof streams run at the least priority, below the MSM tail kernels' streams (msm_scratch_alloc)
        int least = 0, greatest = 0;
        CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
        for (int i = 0; i < NQ; i++) { CUDA_CHECK(cudaStreamCreateWithPriority(&ctx->st[i], cudaStreamNonBlocking, least)); CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming)); }
        CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_w, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_sort, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_pre, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_sortb, cudaEventDisableTiming));
        CUDA_CHECK(cudaStreamCreateWithPriority(&ctx->st_glue, cudaStreamNonBlocking, least));
        for (auto& e : ctx->ev_t) CUDA_CHECK(cudaEventCreate(&e));
        CUDA_CHECK(cudaMalloc(&ctx->d_partial, REC_BYTES));
        CUDA_CHECK(cudaMemset(ctx->d_partial, 0, REC_BYTES));
        CUDA_CHECK(cudaMalloc(&ctx->d_partials_all, 64 * REC_BYTES));
        CUDA_CHECK(cudaMalloc(&ctx->d_proof, 256));
        CUDA_CHECK(cudaMalloc(&ctx->d_pre, PRE_BYTES));
        CUDA_CHECK(cudaMalloc(&ctx->d_rs, 64));
        CUDA_CHECK(cudaMallocHost(&ctx->h_rs, 64));
        CUDA_CHECK(cudaMallocHost(&ctx->h_proof, 256));
        CUDA_CHECK(cudaMalloc(&ctx->d_epoch, 8));
        CUDA_CHECK(cudaMemset(ctx->d_epoch, 0, 8));
        { const char* g = getenv("B2G_GRAPH"); ctx->use_graph = !(g && *g == '0'); }
        // L2 -> DRAM fetch granularity: a 64-byte gather from the fixed-base tables needs only 64 B, so the hint asks for 64 B
        // instead of the device default (128 B); it cut the G1 accumulation's DRAM traffic on the previous target GPU.  On an
        // H100 (700 W, 2^20 chain) it is neutral: 42.2 / 41.8 proofs/s with 64 B vs 41.8 with 128 B, G1 accumulation 2.66-2.68 vs
        // 2.68 ms (DRAM traffic not measured).  Device-wide hint: a failure to set it is ignored.
        cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 64); cudaGetLastError();
        CUDA_CHECK(cudaMalloc(&ctx->d_peer_ptrs, 64 * sizeof(uint8_t*)));
        msm_init_kernels();
        *out = ctx;
    });
}

int b2g_ctx_destroy(b2g_ctx* ctx) {
    return guarded([&] {
        if (!ctx) return;
        DevGuard g(ctx->device);
        cudaDeviceSynchronize();
        for (int i = 0; i < NQ; i++) { if (ctx->scratch_ok) msm_scratch_free(ctx->scratch[i]); cudaStreamDestroy(ctx->st[i]); cudaEventDestroy(ctx->ev_done[i]); }
        cudaEventDestroy(ctx->ev_w); cudaEventDestroy(ctx->ev_sort); cudaEventDestroy(ctx->ev_pre); cudaEventDestroy(ctx->ev_fork); cudaEventDestroy(ctx->ev_sortb); cudaStreamDestroy(ctx->st_glue);
        if (ctx->d_wb) cudaFree(ctx->d_wb);
        for (GraphSlot& s : ctx->graphs) if (s.exec) cudaGraphExecDestroy(s.exec);
        if (ctx->d_keyed) cudaFree(ctx->d_keyed);
        if (ctx->h_rs) cudaFreeHost(ctx->h_rs);
        if (ctx->h_proof) cudaFreeHost(ctx->h_proof);
        if (ctx->d_rs) cudaFree(ctx->d_rs);
        if (ctx->d_epoch) cudaFree(ctx->d_epoch);
        for (auto& e : ctx->ev_t) cudaEventDestroy(e);
        for (int k = 0; k < 64; k++) if (ctx->peer_mapped[k]) cudaIpcCloseMemHandle(ctx->peer_mapped[k]);
        verify_bufs_free(ctx->vbufs);
        for (void* p : {(void*)ctx->d_xchg, (void*)ctx->d_peer_ptrs, (void*)ctx->d_partial, (void*)ctx->d_partials_all, (void*)ctx->d_proof, (void*)ctx->d_pre, (void*)ctx->d_w,
                        (void*)ctx->d_a, (void*)ctx->d_b, (void*)ctx->d_c, (void*)ctx->d_h}) if (p) cudaFree(p);
        delete ctx;
    });
}

int b2g_pk_load(b2g_ctx* ctx, const b2g_pk_desc* d, b2g_pk** out) {
    return guarded([&] {
        if (!ctx || !d || !out) throw_error(B2G_E_SHAPE, "null pointer");
        pk_desc_check(d);
        DevGuard g(ctx->device);
        cudaStream_t st = ctx->st[0];
        // everything allocated below is released if any later step throws (off-curve point, out of memory, ...)
        struct PkGuard {
            b2g_pk* pk = new b2g_pk(); void* tmp = nullptr;
            ~PkGuard() { if (tmp) cudaFree(tmp); if (pk) pk_release(pk); }
        } guard;
        b2g_pk* pk = guard.pk;
        pk->device = ctx->device; pk->shard_rank = ctx->shard_rank; pk->shard_count = ctx->shard_count; pk->n_vars = d->n_vars; pk->n_public = d->n_public; pk->domain = d->domain_size;
        // query sizes as paired with scalars by create_proof_with_assignment (SURVEY.md 3.4)
        const std::vector<uint8_t> l = l_padded(d);
        const uint32_t total[NQ] = {d->domain_size, d->n_vars - 1, d->n_vars - 1, d->n_vars - 1, d->n_vars - 1};
        const uint32_t base_skip[NQ] = {0, 0, 1, 1, 1};             // query[0] is added separately for A/B1/B2
        const uint32_t soff[NQ] = {0, 1, 1, 1, 1};                  // first scalar: h[0] / w[1]
        const void* src[NQ] = {d->h_query, l.data(), d->a_query, d->b_g1_query, d->b_g2_query};
        std::vector<uint32_t> bidx;                                   // real (non-infinity) B bases of this shard, see b2g_pk::d_bidx
        std::vector<uint8_t> bpacked[2];
        for (int q = 0; q < NQ; q++) {
            const bool g2 = q == Q_B2;
            const size_t aff = g2 ? 128 : 64;
            const uint64_t R = ctx->shard_count, r = ctx->shard_rank;
            pk->lo[q] = (uint32_t)((uint64_t)total[q] * r / R);
            pk->cnt[q] = (uint32_t)((uint64_t)total[q] * (r + 1) / R) - pk->lo[q];
            pk->scalar_off[q] = soff[q];
            if (total[q] && !src[q]) throw_error(B2G_E_SHAPE, "null proving-key section");
            if (q == Q_B1 && b_support(d, pk->lo[q], pk->cnt[q], bidx, bpacked)) {
                pk->b_compact = (uint32_t)bidx.size();
                pk->d_bidx = dev_upload<uint32_t>(bidx.data(), bidx.size() * 4, st);
            }
            const bool compact = pk->d_bidx && (q == Q_B1 || q == Q_B2);
            const uint32_t n = compact ? pk->b_compact : pk->cnt[q];
            const void* bases = compact ? (const void*)bpacked[g2 ? 1 : 0].data() : (const uint8_t*)src[q] + (size_t)(base_skip[q] + pk->lo[q]) * aff;
            table_from_host(guard.tmp, bases, n, aff, st, [&](const void* b) { msm_build_table(pk->plan[q], b, n, g2, st); g_launch_count += 1; });
        }
        pk_load_glue(pk, d, st);
        guard.pk = nullptr;
        *out = pk;
    });
}

int b2g_pk_free(b2g_pk* pk) {
    return guarded([&] {
        if (!pk) return;
        DevGuard g(pk->device);
        cudaDeviceSynchronize();
        pk_release(pk);
    });
}

}  // extern "C"
namespace b2g {

int mat_desc_check(const b2g_mat_desc* d, bool with_c) {
    if (!d->a_rowptr || !d->b_rowptr) throw_error(B2G_E_SHAPE, "null row pointer array");
    if (d->num_inputs == 0 || d->num_inputs > d->n_vars) throw_error(B2G_E_SHAPE, "num_inputs out of range");
    const uint64_t need = (uint64_t)d->num_constraints + d->num_inputs;
    int logn = 0;
    while ((1ull << logn) < need) logn++;
    if (logn > 27) throw_error(B2G_E_DOMAIN, "PolynomialDegreeTooLarge: domain (and its double) must fit 2^28");
    const uint32_t m = d->num_constraints;
    const uint32_t annz = d->a_rowptr[m], bnnz = d->b_rowptr[m];
    if ((annz && (!d->a_col || !d->a_val)) || (bnnz && (!d->b_col || !d->b_val))) throw_error(B2G_E_SHAPE, "null matrix arrays");
    if (d->reduction > B2G_REDUCTION_LIBSNARK) throw_error(B2G_E_SHAPE, "unknown reduction");
    const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
    if (with_c && !d->c_rowptr) throw_error(B2G_E_SHAPE, "b2g_setup needs the C matrix (it may have no nonzeros)");
    if (libsnark && !d->c_rowptr) throw_error(B2G_E_SHAPE, "LibsnarkReduction needs the C matrix");
    with_c = with_c || libsnark;
    const uint32_t cnnz = with_c ? d->c_rowptr[m] : 0;
    if (cnnz && (!d->c_col || !d->c_val)) throw_error(B2G_E_SHAPE, "null matrix arrays");
    // row pointers index col / val on the device: must start at 0 and never decrease (the last one is the nnz used above)
    auto check_rowptr = [&](const uint32_t* rp, const char* name) {
        if (rp[0] != 0) throw_error(B2G_E_SHAPE, std::string("matrix ") + name + ": rowptr[0] != 0");
        for (uint32_t i = 0; i < m; i++) if (rp[i + 1] < rp[i]) throw_error(B2G_E_SHAPE, std::string("matrix ") + name + ": row pointers decrease at row " + std::to_string(i));
    };
    check_rowptr(d->a_rowptr, "A"); check_rowptr(d->b_rowptr, "B");
    if (with_c) check_rowptr(d->c_rowptr, "C");
    for (uint32_t k = 0; k < cnnz; k++) if (d->c_col[k] >= d->n_vars) throw_error(B2G_E_SHAPE, "matrix C column index out of range");
    for (uint32_t k = 0; k < annz; k++) if (d->a_col[k] >= d->n_vars) throw_error(B2G_E_SHAPE, "matrix A column index out of range");
    for (uint32_t k = 0; k < bnnz; k++) if (d->b_col[k] >= d->n_vars) throw_error(B2G_E_SHAPE, "matrix B column index out of range");
    return logn;
}

}  // namespace b2g

extern "C" {

static void mat_release(b2g_mat* mat) {
    ntt_domain_destroy(mat->dom);
    for (void* p : {(void*)mat->a_rowptr, (void*)mat->a_col, (void*)mat->b_rowptr, (void*)mat->b_col, (void*)mat->a_val, (void*)mat->b_val,
                    (void*)mat->c_rowptr, (void*)mat->c_col, (void*)mat->c_val}) if (p) cudaFree(p);
    delete mat;
}

int b2g_matrices_load(b2g_ctx* ctx, const b2g_mat_desc* d, b2g_mat** out) {
    return guarded([&] {
        if (!ctx || !d || !out) throw_error(B2G_E_SHAPE, "null pointer");
        const int logn = mat_desc_check(d, false);
        const uint32_t m = d->num_constraints;
        const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
        const uint32_t annz = d->a_rowptr[m], bnnz = d->b_rowptr[m], cnnz = libsnark ? d->c_rowptr[m] : 0;
        DevGuard g(ctx->device);
        cudaStream_t st = ctx->st[0];
        b2g_mat* mat = new b2g_mat();
        struct MatGuard { b2g_mat* m; ~MatGuard() { if (m) { cudaDeviceSynchronize(); mat_release(m); } } } guard{mat};   // a failed upload or table build frees everything
        mat->device = ctx->device; mat->m = m; mat->num_inputs = d->num_inputs; mat->n_vars = d->n_vars; mat->logn = logn; mat->n = 1u << logn;
        mat->a_rowptr = dev_upload<uint32_t>(d->a_rowptr, ((size_t)m + 1) * 4, st);
        mat->b_rowptr = dev_upload<uint32_t>(d->b_rowptr, ((size_t)m + 1) * 4, st);
        mat->a_col = dev_upload<uint32_t>(d->a_col, (size_t)annz * 4, st);
        mat->b_col = dev_upload<uint32_t>(d->b_col, (size_t)bnnz * 4, st);
        mat->a_val = dev_upload<fe>(d->a_val, (size_t)annz * 32, st);
        mat->b_val = dev_upload<fe>(d->b_val, (size_t)bnnz * 32, st);
        mat->reduction = d->reduction;
        if (libsnark) {
            mat->c_rowptr = dev_upload<uint32_t>(d->c_rowptr, ((size_t)m + 1) * 4, st);
            mat->c_col = dev_upload<uint32_t>(d->c_col, (size_t)cnnz * 4, st);
            mat->c_val = dev_upload<fe>(d->c_val, (size_t)cnnz * 32, st);
        }
        ntt_domain_create(mat->dom, logn, st, libsnark);
        g_launch_count += 2;
        CUDA_CHECK(cudaStreamSynchronize(st));
        guard.m = nullptr;
        *out = mat;
    });
}

int b2g_matrices_free(b2g_mat* mat) {
    return guarded([&] {
        if (!mat) return;
        DevGuard g(mat->device);
        cudaDeviceSynchronize();
        mat_release(mat);
    });
}

int b2g_witness_map(b2g_ctx* ctx, b2g_mat* mat, const void* w_mont, void* h_out, uint32_t* domain_size_out) {
    return guarded([&] {
        if (!ctx || !mat || !w_mont) throw_error(B2G_E_SHAPE, "null pointer");
        if (mat->device != ctx->device) throw_error(B2G_E_SHAPE, "handle belongs to another device");
        DevGuard g(ctx->device);
        cudaStream_t st = ctx->st[0];
        ensure_witness_buffers(ctx, mat->n_vars, mat->n);
        CUDA_CHECK(cudaMemcpyAsync(ctx->d_w, w_mont, (size_t)mat->n_vars * 32, cudaMemcpyHostToDevice, st));
        run_witness_map(ctx, mat, st);
        if (h_out) CUDA_CHECK(cudaMemcpyAsync(h_out, ctx->d_h, (size_t)mat->n * 32, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (domain_size_out) *domain_size_out = mat->n;
    });
}

// prologue of the shard entry points (b2g_prove_partial, b2g_prove_sharded_p2p): checks, buffers of one proof, witness upload
static void prove_common(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* w_mont, bool slice_only = false) {
    check_shapes(ctx, pk, mat);
    if (!w_mont) throw_error(B2G_E_SHAPE, "null witness");
    ensure_witness_buffers(ctx, mat->n_vars, mat->n);
    ensure_batch_buffers(ctx, 1);
    ensure_scratch(ctx, pk);
    cudaStream_t s0 = ctx->st[0];
    CUDA_CHECK(cudaEventRecord(ctx->ev_t[12], s0));
    // a rank that takes no part in the split witness map needs only the scalars of its own base range
    size_t first = 0, count = mat->n_vars;
    if (slice_only && map_is_split(ctx, mat) && ctx->shard_rank >= MAP_RANKS) { first = (size_t)pk->scalar_off[Q_A] + pk->lo[Q_A]; count = pk->cnt[Q_A]; }
    if (count) CUDA_CHECK(cudaMemcpyAsync(ctx->d_w + first, (const uint8_t*)w_mont + first * 32, count * 32, cudaMemcpyHostToDevice, s0));
    CUDA_CHECK(cudaEventRecord(ctx->ev_t[13], s0));
}

static double host_ms_since(const std::chrono::steady_clock::time_point& t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// enqueue `count` whole proofs of one circuit (r_j, s_j 32 B apart, witness j at w_mont[j]); nothing here waits for the
// device (the witnesses must be page-locked for the upload to be asynchronous too).  The proof bytes come back through the
// context's own pinned slot; prove_wait copies them to proofs_out.
static void prove_submit(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, uint32_t count, const void* r_canon, const void* s_canon, const void* const* w_mont,
                         uint8_t* proofs_out) {
    if (!ctx || !r_canon || !s_canon || !w_mont || !proofs_out) throw_error(B2G_E_SHAPE, "null pointer");
    if (ctx->shard_count != 1) throw_error(B2G_E_SHAPE, "a whole proof (b2g_prove, b2g_prove_many) needs an unsharded context; use b2g_prove_partial/finish");
    ctx_idle(ctx);
    if (count == 0 || count > MAX_BATCH) throw_error(B2G_E_SHAPE, "b2g_prove_many: count must be in [1, " + std::to_string(MAX_BATCH) + "]");
    for (uint32_t j = 0; j < count; j++) if (!w_mont[j]) throw_error(B2G_E_SHAPE, "null witness " + std::to_string(j));
    const auto t0 = std::chrono::steady_clock::now();
    check_shapes(ctx, pk, mat);
    // the sorted entries and bucket keys of a whole batch are u32 positions into one list
    for (int q = 0; q < NQ; q++) {
        const MsmPlan& p = pk->plan[q];
        if (!p.table) continue;
        if ((uint64_t)count * p.n * p.nwin >= (1ull << 32) || (uint64_t)count * p.nbuckets >= (1ull << 32))
            throw_error(B2G_E_SHAPE, "b2g_prove_many: count x bases x windows of a query reaches 2^32 sorted entries; prove fewer per call");
    }
    prove_pass(ctx, count, 0, true, r_canon, s_canon, w_mont, &mat->n_vars, nullptr,
               [&] {
                   ensure_witness_buffers(ctx, mat->n_vars, mat->n, count);
                   ensure_batch_buffers(ctx, count);
                   ensure_scratch(ctx, pk, count);
               },
               [&] {
                   ctx->last_ms[9] = (float)host_ms_since(t0);
                   run_proof(ctx, pk, mat, 0, count);
               });
    CUDA_CHECK(cudaEventRecord(ctx->ev_t[15], ctx->st[0]));
    ctx->pending_out = proofs_out;
    ctx->pending_count = count;
    ctx->last_ms[10] = (float)host_ms_since(t0);
}

static void prove_wait(b2g_ctx* ctx) {
    if (!ctx) throw_error(B2G_E_SHAPE, "null pointer");
    if (!ctx->pending_out) throw_error(B2G_E_SHAPE, "no submitted proof is pending on this context");
    const auto t0 = std::chrono::steady_clock::now();
    uint8_t* out = ctx->pending_out;
    ctx->pending_out = nullptr;
    CUDA_CHECK(cudaStreamSynchronize(ctx->st[0]));
    memcpy(out, ctx->h_proof, (size_t)ctx->pending_count * 256);
    ctx->last_ms[11] = (float)host_ms_since(t0);
    collect_timings(ctx);
}

int b2g_prove(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont, uint8_t proof_out[256]) {
    return guarded([&] {
        if (!ctx) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        prove_submit(ctx, pk, mat, 1, r_canon, s_canon, &w_mont, proof_out);
        prove_wait(ctx);
    });
}

int b2g_prove_submit(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont, uint8_t proof_out[256]) {
    return guarded([&] {
        if (!ctx) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        prove_submit(ctx, pk, mat, 1, r_canon, s_canon, &w_mont, proof_out);
    });
}

int b2g_prove_many(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, uint32_t count, const void* r_canon, const void* s_canon, const void* const* w_mont,
                   uint8_t* proofs_out) {
    return guarded([&] {
        if (!ctx) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        prove_submit(ctx, pk, mat, count, r_canon, s_canon, w_mont, proofs_out);
        prove_wait(ctx);
    });
}

int b2g_host_register(const void* ptr, size_t bytes) {
    return guarded([&] {
        if (!ptr || !bytes) throw_error(B2G_E_SHAPE, "null pointer");
        cudaError_t e = cudaHostRegister(const_cast<void*>(ptr), bytes, cudaHostRegisterDefault);
        if (e != cudaSuccess && e != cudaErrorHostMemoryAlreadyRegistered) CUDA_CHECK(e);
        cudaGetLastError();
    });
}

int b2g_host_unregister(const void* ptr) {
    return guarded([&] {
        if (!ptr) throw_error(B2G_E_SHAPE, "null pointer");
        cudaError_t e = cudaHostUnregister(const_cast<void*>(ptr));
        if (e != cudaSuccess && e != cudaErrorHostMemoryNotRegistered) CUDA_CHECK(e);
        cudaGetLastError();
    });
}

int b2g_prove_wait(b2g_ctx* ctx) {
    return guarded([&] {
        if (!ctx) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        prove_wait(ctx);
    });
}

int b2g_prove_partial(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont, void* partial_out) {
    return guarded([&] {
        if (!ctx || !pk || !partial_out) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        ctx->pre_valid = false;
        prove_common(ctx, pk, mat, w_mont);
        if (r_canon && s_canon) { stage_rs(ctx, r_canon, s_canon); launch_glue_pre(ctx, pk); }
        launch_msms(ctx, pk, mat, true, false);
        cudaStream_t s0 = ctx->st[0];
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[14], s0));
        CUDA_CHECK(cudaMemcpyAsync(partial_out, ctx->d_partial, B2G_PARTIAL_BYTES, cudaMemcpyDeviceToHost, s0));
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[15], s0));
        CUDA_CHECK(cudaStreamSynchronize(s0));
        collect_timings(ctx);
    });
}

int b2g_prove_finish(b2g_ctx* ctx, b2g_pk* pk, const void* partials_all, int count, const void* r_canon, const void* s_canon, uint8_t proof_out[256]) {
    return guarded([&] {
        if (!ctx || !pk || !partials_all || !r_canon || !s_canon || !proof_out) throw_error(B2G_E_SHAPE, "null pointer");
        if (count < 1 || count > 64) throw_error(B2G_E_SHAPE, "partial count out of range");
        check_pk_ctx(ctx, pk);
        DevGuard g(ctx->device);
        ensure_batch_buffers(ctx, 1);
        cudaStream_t s0 = ctx->st[0];
        if (!(ctx->pre_valid && !memcmp(ctx->pre_r, r_canon, 32) && !memcmp(ctx->pre_s, s_canon, 32))) { stage_rs(ctx, r_canon, s_canon); launch_glue_pre(ctx, pk); }
        ctx->pre_valid = false;
        // the records the peer-memory gather writes: each rank's partial, then s*A_k and r*B1_k (all ranks share one (r, s)),
        // the two products side by side on the A and B1 streams
        CUDA_CHECK(cudaMemcpy2DAsync(ctx->d_partials_all, REC_BYTES, partials_all, B2G_PARTIAL_BYTES, B2G_PARTIAL_BYTES, count, cudaMemcpyHostToDevice, s0));
        CUDA_CHECK(cudaEventRecord(ctx->ev_fork, s0));
        const Scalar256* rs = reinterpret_cast<const Scalar256*>(ctx->d_rs);
        for (int q : {Q_A, Q_B1}) {
            CUDA_CHECK(cudaStreamWaitEvent(ctx->st[q], ctx->ev_fork, 0));
            scale_partial_kernel<<<count, 32, 0, ctx->st[q]>>>(ctx->d_partials_all + PARTIAL_OFF[q], q == Q_A ? rs + 1 : rs, ctx->d_partials_all + B2G_PARTIAL_BYTES + (q == Q_A ? 0 : 128), 0);
            CUDA_CHECK(cudaEventRecord(ctx->ev_done[q], ctx->st[q]));
            CUDA_CHECK(cudaStreamWaitEvent(s0, ctx->ev_done[q], 0));
        }
        g_launch_count += 2;
        launch_glue_post(ctx, pk, ctx->d_partials_all, count, s0);
        CUDA_CHECK(cudaMemcpyAsync(proof_out, ctx->d_proof, 256, cudaMemcpyDeviceToHost, s0));
        CUDA_CHECK(cudaStreamSynchronize(s0));
    });
}

int b2g_ctx_prepare(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat) {
    return guarded([&] {
        check_shapes(ctx, pk, mat);
        DevGuard g(ctx->device);
        ensure_witness_buffers(ctx, mat->n_vars, mat->n);
        ensure_scratch(ctx, pk);
        CUDA_CHECK(cudaDeviceSynchronize());
    });
}

}  // extern "C"
// the arena is sized for the largest domain this context has been prepared for (b2g_ctx_prepare / a first proof): call that
// BEFORE wiring the peers, or the witness map stays replicated on every rank
static void ensure_arena(b2g_ctx* ctx) {
    if (ctx->d_xchg) return;
    ctx->eval_cap = ctx->cap_n;
    const size_t bytes = EVAL_OFF + ctx->eval_cap * sizeof(fe);
    CUDA_CHECK(cudaMalloc(&ctx->d_xchg, bytes));                       // plain cudaMalloc: exportable through CUDA IPC
    CUDA_CHECK(cudaMemset(ctx->d_xchg, 0, EVAL_OFF));
}
extern "C" {

int b2g_p2p_export(b2g_ctx* ctx, void* handle_out) {
    return guarded([&] {
        if (!ctx || !handle_out) throw_error(B2G_E_SHAPE, "null pointer");
        static_assert(sizeof(cudaIpcMemHandle_t) + 16 == B2G_IPC_HANDLE_BYTES, "IPC handle size");
        DevGuard g(ctx->device);
        ensure_arena(ctx);
        cudaIpcMemHandle_t h;
        CUDA_CHECK(cudaIpcGetMemHandle(&h, ctx->d_xchg));
        memset(handle_out, 0, B2G_IPC_HANDLE_BYTES);
        memcpy(handle_out, &h, sizeof h);
        const uint64_t cap = ctx->eval_cap;
        memcpy((uint8_t*)handle_out + sizeof h, &cap, 8);
    });
}

int b2g_p2p_import(b2g_ctx* ctx, const void* handles_all, int count) {
    return guarded([&] {
        if (!ctx || !handles_all) throw_error(B2G_E_SHAPE, "null pointer");
        if (count != ctx->shard_count) throw_error(B2G_E_SHAPE, "need one handle per shard rank");
        DevGuard g(ctx->device);
        ensure_arena(ctx);
        std::vector<uint8_t*> ptrs((size_t)count, nullptr);
        uint64_t common = ctx->eval_cap;
        for (int k = 0; k < count; k++) {
            const uint8_t* rec = (const uint8_t*)handles_all + (size_t)k * B2G_IPC_HANDLE_BYTES;
            uint64_t cap = 0; memcpy(&cap, rec + sizeof(cudaIpcMemHandle_t), 8);
            if (k != ctx->shard_rank && cap < common) common = cap;
        }
        ctx->eval_common = (size_t)common;
        for (int k = 0; k < count; k++) {
            if (k == ctx->shard_rank) { ptrs[k] = ctx->d_xchg; continue; }
            cudaIpcMemHandle_t h; memcpy(&h, (const uint8_t*)handles_all + (size_t)k * B2G_IPC_HANDLE_BYTES, sizeof h);
            void* p = nullptr;
            CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
            ctx->peer_mapped[k] = p; ptrs[k] = (uint8_t*)p;
        }
        CUDA_CHECK(cudaMemcpy(ctx->d_peer_ptrs, ptrs.data(), (size_t)count * sizeof(uint8_t*), cudaMemcpyHostToDevice));
        ctx->peers_imported = count; ctx->alloc_gen++;          // captured graphs were built without the peers
    });
}

int b2g_p2p_connect_local(b2g_ctx** ctxs, int count) {
    return guarded([&] {
        if (!ctxs || count < 1 || count > 64) throw_error(B2G_E_SHAPE, "bad arguments");
        for (int k = 0; k < count; k++) if (!ctxs[k] || ctxs[k]->shard_rank != k || ctxs[k]->shard_count != count) throw_error(B2G_E_SHAPE, "contexts must be the shard ranks 0..count-1 in order");
        std::vector<uint8_t*> ptrs((size_t)count);
        size_t common = (size_t)-1;
        for (int k = 0; k < count; k++) { DevGuard g(ctxs[k]->device); ensure_arena(ctxs[k]); ptrs[k] = ctxs[k]->d_xchg; common = std::min(common, ctxs[k]->eval_cap); }
        for (int k = 0; k < count; k++) ctxs[k]->eval_common = common;
        for (int k = 0; k < count; k++) {
            DevGuard g(ctxs[k]->device);
            for (int j = 0; j < count; j++) if (ctxs[j]->device != ctxs[k]->device) {
                cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[j]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CUDA_CHECK(e);
                cudaGetLastError();
            }
            CUDA_CHECK(cudaMemcpy(ctxs[k]->d_peer_ptrs, ptrs.data(), (size_t)count * sizeof(uint8_t*), cudaMemcpyHostToDevice));
            ctxs[k]->peers_imported = count; ctxs[k]->alloc_gen++;
        }
    });
}

int b2g_prove_sharded_p2p(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, const void* r_canon, const void* s_canon, const void* w_mont, uint8_t proof_out[256]) {
    return guarded([&] {
        if (!ctx || !pk || !r_canon || !s_canon || !proof_out) throw_error(B2G_E_SHAPE, "null pointer");
        if (ctx->peers_imported != ctx->shard_count) throw_error(B2G_E_SHAPE, "b2g_p2p_import has not been called with every rank's handle");
        DevGuard g(ctx->device);
        prove_common(ctx, pk, mat, w_mont, true);
        stage_rs(ctx, r_canon, s_canon);
        cudaStream_t s0 = ctx->st[0];
        run_proof(ctx, pk, mat, 1);
        ctx->pre_valid = false;
        unsigned int* d_flag = reinterpret_cast<unsigned int*>(ctx->d_xchg + XCHG_BYTES);
        unsigned int flag = 0;
        CUDA_CHECK(cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, s0));
        CUDA_CHECK(cudaMemcpyAsync(proof_out, ctx->d_proof, 256, cudaMemcpyDeviceToHost, s0));
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[15], s0));
        CUDA_CHECK(cudaStreamSynchronize(s0));
        if (flag) throw_error(B2G_E_DEVICE, "peer exchange timed out waiting for shard rank " + std::to_string(flag - 1));
        collect_timings(ctx);
    });
}

int b2g_bench_device(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int iters, float* avg_ms) {
    return guarded([&] {
        if (!avg_ms || iters == 0) throw_error(B2G_E_SHAPE, "bad arguments");
        const bool no_wait = iters < 0;                                   // enqueue only: the caller synchronises and times the window
        if (no_wait) iters = -iters;
        check_shapes(ctx, pk, mat);
        if (ctx->cap_w < mat->n_vars) throw_error(B2G_E_SHAPE, "no witness resident: call b2g_prove first");
        DevGuard g(ctx->device);
        ensure_scratch(ctx, pk);
        cudaStream_t s0 = ctx->st[0];
        // representative full-size scalars (the glue cost depends on their bit length)
        Scalar256 kr = {{0x90abcdefu, 0x12345678u, 0x90abcdefu, 0x12345678u, 0x0badc0deu, 0x0defaced, 0x13572468u, 0x1fedcba9u}};
        Scalar256 ks = {{0x87654321u, 0xfedcba09u, 0x87654321u, 0xfedcba09u, 0x600dcafeu, 0x0ddba11u, 0x24681357u, 0x2abcdef0u}};
        stage_rs(ctx, kr.l, ks.l);
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[16], s0));
        for (int it = 0; it < iters; it++) run_proof(ctx, pk, mat, 0);
        ctx->pre_valid = false;
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[17], s0));
        if (no_wait) { *avg_ms = 0.f; return; }
        CUDA_CHECK(cudaStreamSynchronize(s0));
        float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->ev_t[16], ctx->ev_t[17]));
        *avg_ms = ms / iters;
    });
}

int b2g_bench_msm(b2g_ctx* ctx, b2g_pk* pk, b2g_mat* mat, int query, int iters, float out_ms[2]) {
    return guarded([&] {
        if (!out_ms || iters < 1 || query < 0 || query >= NQ) throw_error(B2G_E_SHAPE, "bad arguments");
        check_shapes(ctx, pk, mat);
        if (ctx->cap_w < mat->n_vars) throw_error(B2G_E_SHAPE, "no witness resident: call b2g_prove first");
        DevGuard g(ctx->device);
        cudaStream_t s0 = ctx->st[0];
        MsmScratch& sc = ctx->scratch[query];
        const bool on_b = pk->d_bidx && (query == Q_B1 || query == Q_B2);      // sparse B: compacted scalars of the last proof
        MsmScratch& sorter = ctx->scratch[query == Q_H ? Q_H : (on_b ? Q_B1 : Q_L)];
        const fe* scalars = on_b ? ctx->d_wb : (query == Q_H ? ctx->d_h : ctx->d_w + pk->scalar_off[query]) + pk->lo[query];
        const uint32_t nscal = on_b ? pk->b_compact : pk->cnt[query];
        std::vector<cudaEvent_t> ev(2 * (size_t)iters);
        for (auto& e : ev) CUDA_CHECK(cudaEventCreate(&e));
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[18], s0));
        for (int it = 0; it < iters; it++) {
            sc.prof0 = ev[2 * it]; sc.prof1 = ev[2 * it + 1];
            msm_sort(pk->plan[query], sorter, scalars, nscal, true, s0);
            msm_accumulate(pk->plan[query], sorter, sc, s0);
        }
        sc.prof0 = sc.prof1 = nullptr;
        CUDA_CHECK(cudaEventRecord(ctx->ev_t[19], s0));
        CUDA_CHECK(cudaStreamSynchronize(s0));
        float total = 0, acc = 0;
        CUDA_CHECK(cudaEventElapsedTime(&total, ctx->ev_t[18], ctx->ev_t[19]));
        for (int it = 0; it < iters; it++) { float ms = 0; cudaEventElapsedTime(&ms, ev[2 * it], ev[2 * it + 1]); acc += ms; }
        for (auto& e : ev) cudaEventDestroy(e);
        out_ms[0] = total / iters; out_ms[1] = acc / iters;
    });
}

int b2g_last_timings(b2g_ctx* ctx, float out_ms[16]) {
    return guarded([&] { if (!ctx || !out_ms) throw_error(B2G_E_SHAPE, "null pointer"); memcpy(out_ms, ctx->last_ms, sizeof(ctx->last_ms)); });
}

int b2g_launch_count(b2g_ctx* ctx, uint64_t* count) {
    return guarded([&] { if (!ctx || !count) throw_error(B2G_E_SHAPE, "null pointer"); *count = g_launch_count.load(); });
}

// ---------------------------------------------------------------------------------------- kernel-level entry points
}  // extern "C"
template <bool IS_G2>
static void msm_entry(b2g_ctx* ctx, const void* bases, const void* scalars, size_t n, int scalars_mont, void* out) {
    if (!ctx || !out || (n && (!bases || !scalars))) throw_error(B2G_E_SHAPE, "null pointer");
    if (n >= (1ull << 27)) throw_error(B2G_E_SHAPE, "msm too large");
    DevGuard g(ctx->device);
    cudaStream_t st = ctx->st[0];
    const size_t aff = IS_G2 ? 128 : 64, ptb = 2 * aff;
    if (n == 0) { memset(out, 0, aff); return; }
    uint8_t* d_bases = dev_upload<uint8_t>(bases, n * aff, st);
    fe* d_sc = dev_upload<fe>(scalars, n * 32, st);
    MsmPlan plan; MsmScratch sc;
    msm_build_table(plan, d_bases, (uint32_t)n, IS_G2, st);
    msm_scratch_alloc(sc, (uint32_t)n, plan.nwin, plan.nbuckets, IS_G2, true);
    msm_run(plan, sc, d_sc, (uint32_t)n, scalars_mont != 0, st);
    uint8_t* d_out = nullptr; CUDA_CHECK(cudaMalloc(&d_out, aff));
    if (IS_G2) xyzz_to_affine_kernel<G2, Fq2><<<1, 1, 0, st>>>(sc.result, 1, d_out);
    else xyzz_to_affine_kernel<G1, Fq><<<1, 1, 0, st>>>(sc.result, 1, d_out);
    g_launch_count += 2;
    CUDA_CHECK(cudaMemcpyAsync(out, d_out, aff, cudaMemcpyDeviceToHost, st));
    cudaError_t e = cudaStreamSynchronize(st);
    (void)ptb;
    cudaFree(d_out); cudaFree(d_bases); cudaFree(d_sc); msm_free_table(plan); msm_scratch_free(sc);
    CUDA_CHECK(e);
}

extern "C" {
int b2g_msm_g1(b2g_ctx* ctx, const void* bases, const void* scalars, size_t n, int scalars_mont, void* out) {
    return guarded([&] { msm_entry<false>(ctx, bases, scalars, n, scalars_mont, out); });
}
int b2g_msm_g2(b2g_ctx* ctx, const void* bases, const void* scalars, size_t n, int scalars_mont, void* out) {
    return guarded([&] { msm_entry<true>(ctx, bases, scalars, n, scalars_mont, out); });
}

int b2g_ntt(b2g_ctx* ctx, void* data, int log_n, int inverse) {
    return guarded([&] {
        if (!ctx || !data) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(ctx->device);
        cudaStream_t st = ctx->st[0];
        NttDomain dom;
        ntt_domain_create(dom, log_n, st);
        const size_t bytes = ((size_t)1 << log_n) * 32;
        fe* d = dev_upload<fe>(data, bytes, st);
        fe* tmp = nullptr; CUDA_CHECK(cudaMalloc(&tmp, bytes));
        ntt_plain(dom, d, tmp, inverse != 0, st);
        CUDA_CHECK(cudaMemcpyAsync(data, d, bytes, cudaMemcpyDeviceToHost, st));
        cudaError_t e = cudaStreamSynchronize(st);
        cudaFree(d); cudaFree(tmp); ntt_domain_destroy(dom);
        CUDA_CHECK(e);
    });
}

}  // extern "C"
template <class C, class F>
static void fixed_base_entry(b2g_ctx* ctx, const void* scalars, size_t n, void* out) {
    if (!ctx || (n && (!scalars || !out))) throw_error(B2G_E_SHAPE, "null pointer");
    if (n == 0) return;
    DevGuard g(ctx->device);
    cudaStream_t st = ctx->st[0];
    const size_t aff = 2 * Bytes<F>::ELEM;
    void* table = nullptr; CUDA_CHECK(cudaMalloc(&table, 32 * 255 * aff));
    fixed_table_kernel<C, F><<<(32 * 255 + 63) / 64, 64, 0, st>>>(table, nullptr);
    const size_t CH = 1u << 22;                                        // bound temporary device memory
    fe* d_sc = nullptr; uint8_t* d_out = nullptr;
    CUDA_CHECK(cudaMalloc(&d_sc, (n < CH ? n : CH) * 32)); CUDA_CHECK(cudaMalloc(&d_out, (n < CH ? n : CH) * aff));
    cudaError_t e = cudaSuccess;
    for (size_t off = 0; off < n && e == cudaSuccess; off += CH) {
        const size_t cnt = n - off < CH ? n - off : CH;
        cudaMemcpyAsync(d_sc, (const uint8_t*)scalars + off * 32, cnt * 32, cudaMemcpyHostToDevice, st);
        fixed_base_kernel<C, F><<<(unsigned)((cnt + 127) / 128), 128, 0, st>>>(table, d_sc, (uint32_t)cnt, d_out);
        g_launch_count += 1;
        cudaMemcpyAsync((uint8_t*)out + off * aff, d_out, cnt * aff, cudaMemcpyDeviceToHost, st);
        e = cudaStreamSynchronize(st);
    }
    cudaFree(table); cudaFree(d_sc); cudaFree(d_out);
    CUDA_CHECK(e);
}

extern "C" {
int b2g_fixed_base_g1(b2g_ctx* ctx, const void* scalars_canon, size_t n, void* out) {
    return guarded([&] { fixed_base_entry<G1, Fq>(ctx, scalars_canon, n, out); });
}
int b2g_fixed_base_g2(b2g_ctx* ctx, const void* scalars_canon, size_t n, void* out) {
    return guarded([&] { fixed_base_entry<G2, Fq2>(ctx, scalars_canon, n, out); });
}

int b2g_test_op(b2g_ctx* ctx, int op, const void* a, const void* b, size_t n, void* out) {
    return guarded([&] {
        if (ctx && op == SCALE_SPLIT_TEST_OP) { DevGuard g(ctx->device); scale_split_test_op(ctx->st[0], a, n, out); return; }
        if (ctx && op >= PAIRING_TEST_OP0) { DevGuard g(ctx->device); pairing_test_op(ctx->st[0], op, a, b, n, out); return; }
        TestOpShape s;
        if (!ctx || !a || !out || !test_op_shape(op, s)) throw_error(B2G_E_SHAPE, "bad arguments");
        if (!b && s.b && s.b != s.a) throw_error(B2G_E_SHAPE, "this op needs operand b");
        if (n == 0) return;
        DevGuard g(ctx->device);
        cudaStream_t st = ctx->st[0];
        uint8_t* da = dev_upload<uint8_t>(a, n * s.a, st);
        uint8_t* db = s.b ? dev_upload<uint8_t>(b ? b : a, n * s.b, st) : nullptr;
        uint8_t* dout = nullptr; CUDA_CHECK(cudaMalloc(&dout, n * s.out));
        const size_t threads = n * s.threads;
        test_op_kernel<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(op, da, db, (uint32_t)n, dout);
        g_launch_count += 1;
        CUDA_CHECK(cudaMemcpyAsync(out, dout, n * s.out, cudaMemcpyDeviceToHost, st));
        cudaError_t e = cudaStreamSynchronize(st);
        cudaFree(da); if (db) cudaFree(db); cudaFree(dout);
        CUDA_CHECK(e);
    });
}

}  // extern "C"

// ================================================================================================== keyed batches
namespace b2g {

static const char* const QUERY_NAME[NQ] = {"H", "L", "A", "B1", "B2"};
// the three sorts of a keyed pass: H over h, W over w[1..] (its entries serve L and A), B over the gathered B scalars (B1 and B2)
enum { S_H = 0, S_W = 1, S_B = 2, NS = 3 };
static const int SORT_QUERY[NS] = {Q_H, Q_A, Q_B1};

// one key's base count per query: H the domain, L and A n_vars - 1, B1 and B2 n_vars - 1 or the count of its real B bases
using KeyBases = std::array<uint32_t, NQ>;

// the window size of each query (msm_pick_c on its largest base count in the group) and each key's first arena row
struct GroupLayout {
    int c[NQ] = {};
    uint64_t rows[NQ] = {};
    std::vector<uint32_t> row[NQ];
};

static GroupLayout group_layout(const std::vector<KeyBases>& bases) {
    if (bases.empty()) throw_error(B2G_E_SHAPE, "b2g_pk_group_load: the group has no keys");
    GroupLayout L;
    for (int q = 0; q < NQ; q++) {
        uint32_t most = 0;
        for (const KeyBases& b : bases) most = std::max(most, b[q]);
        L.c[q] = msm_pick_c(most ? most : 1);
        const int nwin = msm_nwin(L.c[q]);
        for (const KeyBases& b : bases) {
            L.row[q].push_back((uint32_t)L.rows[q]);
            L.rows[q] += (uint64_t)b[q] * nwin;
            // an entry word is a table row with the sign in bit 31
            if (L.rows[q] >= (1ull << 31))
                throw_error(B2G_E_SHAPE, std::string("b2g_pk_group_load: the tables of query ") + QUERY_NAME[q] +
                                         " reach 2^31 rows (the sign bit of an entry word); load fewer or smaller keys per group");
        }
    }
    return L;
}

// the per-proof tables of one call: rows [S_H | S_W | S_B] x count, the key of every proof, and where each key's witnesses
// (n_vars apart) and witness-map vectors (its domain apart) start in the call's buffers; proofs come key after key
struct CallLayout {
    uint32_t count = 0;
    std::vector<KeyedRow> rows;
    std::vector<uint32_t> key_of;
    uint32_t max_n[NS] = {};
    uint64_t total_n[NS] = {};
    std::vector<uint64_t> w_off, v_off;
    uint64_t total_w = 0, total_v = 0;
};

static CallLayout call_layout(const GroupLayout& G, const std::vector<KeyBases>& bases, const std::vector<uint32_t>& n_vars,
                              const std::vector<uint32_t>& n_dom, const uint32_t* counts) {
    const size_t K = bases.size();
    uint64_t total = 0;
    for (size_t k = 0; k < K; k++) total += counts[k];
    if (total == 0 || total > MAX_BATCH) throw_error(B2G_E_SHAPE, "b2g_prove_keys: the total count must be in [1, " + std::to_string(MAX_BATCH) + "]");
    CallLayout C;
    C.count = (uint32_t)total;
    C.rows.resize((size_t)NS * total);
    for (size_t k = 0; k < K; k++) {
        C.w_off.push_back(C.total_w); C.v_off.push_back(C.total_v);
        for (uint32_t i = 0; i < counts[k]; i++) {
            const uint32_t j = (uint32_t)C.key_of.size();
            C.key_of.push_back((uint32_t)k);
            const uint64_t src[NS] = {C.total_v, C.total_w + 1, C.total_n[S_B]};      // h[0], w[1], the gathered B scalars
            for (int t = 0; t < NS; t++) {
                const int q = SORT_QUERY[t];
                C.rows[(size_t)t * total + j] = {src[t], C.total_n[t], bases[k][q], G.row[q][k]};
                C.total_n[t] += bases[k][q];
                C.max_n[t] = std::max(C.max_n[t], bases[k][q]);
            }
            C.total_w += n_vars[k]; C.total_v += n_dom[k];
        }
    }
    // the sorted entries and bucket keys of the whole call are u32 positions into one list
    for (int t = 0; t < NS; t++) {
        const int q = SORT_QUERY[t];
        if (C.total_n[t] * (uint64_t)msm_nwin(G.c[q]) >= (1ull << 32) || total << (G.c[q] - 1) >= (1ull << 32))
            throw_error(B2G_E_SHAPE, std::string("b2g_prove_keys: proofs x bases x windows of query ") + QUERY_NAME[q] +
                                     " reach 2^32 sorted entries; prove fewer per call");
    }
    return C;
}

static void group_release(b2g_pk_group* g) {
    for (b2g_pk* pk : g->keys) pk_release(pk);
    for (int q = 0; q < NQ; q++) msm_free_table(g->plan[q]);
    if (g->d_keys) cudaFree(g->d_keys);
    if (g->d_bidx) cudaFree(g->d_bidx);
    if (g->d_consts) cudaFree(g->d_consts);
    delete g;
}

static std::vector<KeyBases> group_bases(const b2g_pk_group* g) {
    std::vector<KeyBases> b;
    for (const b2g_pk* pk : g->keys) b.push_back({pk->plan[Q_H].n, pk->plan[Q_L].n, pk->plan[Q_A].n, pk->plan[Q_B1].n, pk->plan[Q_B2].n});
    return b;
}

// the rows and key_of of a call, in one device buffer the captured pass points into
static void ensure_keyed_buffer(b2g_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->cap_keyed) return;
    CUDA_CHECK(cudaDeviceSynchronize());
    if (ctx->d_keyed) cudaFree(ctx->d_keyed);
    ctx->d_keyed = nullptr; ctx->cap_keyed = 0; ctx->alloc_gen++;
    CUDA_CHECK(cudaMalloc(&ctx->d_keyed, bytes));
    ctx->cap_keyed = bytes;
}

// The keyed pass, launched as launch_msms + the glue launch a batch of one key: glue_pre on the side stream; the W sort on
// the L stream and, when some key's B query is sparse, the B gather and sort on the B1 stream, both from the witnesses; the
// A, B1, B2, L accumulations on their streams (A and B1 followed by s*A, r*B1); on stream 0 the witness map of every key
// with proofs, then the H sort and accumulation; the assembly once everything is in.
static void enqueue_keys(b2g_ctx* ctx, b2g_pk_group* g, const CallLayout& C, const uint32_t* counts) {
    cudaStream_t s0 = ctx->st[0], ssort = ctx->st[Q_L], sb = ctx->st[Q_B1];
    const uint32_t count = C.count;
    const KeyedRow* rows = reinterpret_cast<const KeyedRow*>(ctx->d_keyed);
    const uint32_t* key_of = reinterpret_cast<const uint32_t*>(rows + (size_t)NS * count);
    fork_glue_pre(ctx, [&](cudaStream_t sg) {
        glue_pre_keys_kernel<<<count, 160, 0, sg>>>(g->d_keys, key_of, reinterpret_cast<const Scalar256*>(ctx->d_rs), ctx->d_pre);
    });
    CUDA_CHECK(cudaEventRecord(ctx->ev_w, s0));
    CUDA_CHECK(cudaStreamWaitEvent(ssort, ctx->ev_w, 0));
    msm_sort_keyed(g->plan[Q_A], ctx->scratch[Q_L], ctx->d_w, true, rows + (size_t)S_W * count, count, C.max_n[S_W], C.total_n[S_W], ssort);
    CUDA_CHECK(cudaEventRecord(ctx->ev_sort, ssort));
    if (g->b_sparse) {
        CUDA_CHECK(cudaStreamWaitEvent(sb, ctx->ev_w, 0));
        if (C.total_n[S_B]) {
            gather_scalars_keyed_kernel<<<dim3((C.max_n[S_B] + 255) / 256, count), 256, 0, sb>>>(ctx->d_w, rows + (size_t)S_W * count, rows + (size_t)S_B * count,
                                                                                                   key_of, g->d_bidx, ctx->d_wb);
            g_launch_count += 1;
        }
        msm_sort_keyed(g->plan[Q_B1], ctx->scratch[Q_B1], ctx->d_wb, true, rows + (size_t)S_B * count, count, C.max_n[S_B], C.total_n[S_B], sb);
        CUDA_CHECK(cudaEventRecord(ctx->ev_sortb, sb));
    }
    // with no sparse key, the B queries have the W sort's base counts, window size and arena rows: they read its entries
    accumulate_witness_queries(ctx, g->plan, g->b_sparse, count, false, true);
    for (size_t k = 0; k < g->keys.size(); k++)
        if (counts[k]) run_witness_map(ctx, g->mats[k], s0, counts[k], C.w_off[k], C.v_off[k]);
    msm_sort_keyed(g->plan[Q_H], ctx->scratch[Q_H], ctx->d_h, true, rows, count, C.max_n[S_H], C.total_n[S_H], s0);
    msm_accumulate(g->plan[Q_H], ctx->scratch[Q_H], ctx->scratch[Q_H], s0);
    for (int q = 1; q < NQ; q++) CUDA_CHECK(cudaStreamWaitEvent(s0, ctx->ev_done[q], 0));
    join_glue_post(ctx, s0, [&] { glue_post_keys_kernel<<<count, 96, 0, s0>>>(ctx->d_partial, g->d_consts, key_of, ctx->d_pre, ctx->d_proof); });
}

}  // namespace b2g

extern "C" {

int b2g_pk_group_load(b2g_ctx* ctx, uint32_t n_keys, const b2g_pk_desc* pks, b2g_mat* const* mats, b2g_pk_group** out) {
    return guarded_clear([&] {
        if (!ctx || !out || (n_keys && (!pks || !mats))) throw_error(B2G_E_SHAPE, "null pointer");
        if (n_keys == 0) throw_error(B2G_E_SHAPE, "b2g_pk_group_load: the group has no keys");
        if (ctx->shard_count != 1) throw_error(B2G_E_SHAPE, "b2g_pk_group_load: a key group needs an unsharded context");
        // every key against its matrices, and the arena rows, before anything is allocated
        std::vector<KeyBases> bases(n_keys);
        std::vector<std::vector<uint32_t>> bidx(n_keys);
        std::vector<std::array<std::vector<uint8_t>, 2>> bpacked(n_keys);
        std::vector<char> sparse(n_keys, 0);
        for (uint32_t k = 0; k < n_keys; k++) {
            const b2g_pk_desc* d = &pks[k];
            try {
                pk_desc_check(d);
                b2g_pk hdr;
                hdr.device = ctx->device; hdr.n_vars = d->n_vars; hdr.n_public = d->n_public; hdr.domain = d->domain_size;
                check_shapes(ctx, &hdr, mats[k]);
            } catch (const B2gError& e) { throw_error(e.code, "b2g_pk_group_load: key " + std::to_string(k) + ": " + e.what()); }
            const uint32_t nw = d->n_vars - 1;
            sparse[k] = b_support(d, 0, nw, bidx[k], bpacked[k].data());
            const uint32_t nb = sparse[k] ? (uint32_t)bidx[k].size() : nw;
            bases[k] = {d->domain_size, nw, nw, nb, nb};
        }
        const GroupLayout L = group_layout(bases);
        DevGuard dg(ctx->device);
        cudaStream_t st = ctx->st[0];
        struct GroupGuard {
            b2g_pk_group* g = new b2g_pk_group(); void* tmp = nullptr;
            ~GroupGuard() { if (tmp) cudaFree(tmp); if (g) { cudaDeviceSynchronize(); group_release(g); } }
        } guard;
        b2g_pk_group* g = guard.g;
        g->device = ctx->device;
        g->mats.assign(mats, mats + n_keys);
        g->b_sparse = std::find(sparse.begin(), sparse.end(), 1) != sparse.end();
        for (int q = 0; q < NQ; q++) {
            MsmPlan& p = g->plan[q];
            p.g2 = q == Q_B2; p.c = L.c[q]; p.nwin = msm_nwin(p.c); p.nbuckets = 1u << (p.c - 1); p.n = 0;
            for (const KeyBases& b : bases) p.n = std::max(p.n, b[q]);
            g->row[q] = L.row[q];
            if (!L.rows[q]) continue;
            const size_t bytes = L.rows[q] * (p.g2 ? 128 : 64);
            if (cudaMalloc(&p.table, bytes) != cudaSuccess) {
                cudaGetLastError(); p.table = nullptr;
                throw_error(B2G_E_DEVICE, std::string("b2g_pk_group_load: the table arena of query ") + QUERY_NAME[q] + " (" +
                                          std::to_string(bytes >> 20) + " MiB for " + std::to_string(n_keys) + " keys) does not fit in device memory");
            }
        }
        std::vector<KeyGlue> glue(n_keys);
        std::vector<const uint32_t*> bidx_dev(n_keys, nullptr);
        std::vector<const uint8_t*> consts_dev(n_keys, nullptr);
        for (uint32_t k = 0; k < n_keys; k++) {
            const b2g_pk_desc* d = &pks[k];
            b2g_pk* pk = new b2g_pk();
            g->keys.push_back(pk);
            pk->device = ctx->device; pk->n_vars = d->n_vars; pk->n_public = d->n_public; pk->domain = d->domain_size;
            try {
                // the bases of each query as b2g_pk_load pairs them with scalars
                const std::vector<uint8_t> l = l_padded(d);
                const void* src[NQ] = {d->h_query, l.data(), (const uint8_t*)d->a_query + 64,
                                       sparse[k] ? (const void*)bpacked[k][0].data() : (const uint8_t*)d->b_g1_query + 64,
                                       sparse[k] ? (const void*)bpacked[k][1].data() : (const uint8_t*)d->b_g2_query + 128};
                for (int q = 0; q < NQ; q++) {
                    pk->plan[q].n = bases[k][q]; pk->plan[q].g2 = q == Q_B2;
                    pk->cnt[q] = q == Q_H ? d->domain_size : d->n_vars - 1;
                    pk->scalar_off[q] = q == Q_H ? 0 : 1;
                    if (!bases[k][q]) continue;
                    const size_t aff = q == Q_B2 ? 128 : 64;
                    table_from_host(guard.tmp, src[q], bases[k][q], aff, st, [&](const void* b) {
                        msm_build_table_into((uint8_t*)g->plan[q].table + (size_t)L.row[q][k] * aff, b, bases[k][q], L.c[q], q == Q_B2, st);
                    });
                }
                if (sparse[k]) {
                    pk->b_compact = bases[k][Q_B1];
                    pk->d_bidx = dev_upload<uint32_t>(bidx[k].data(), bidx[k].size() * 4, st);
                }
                pk_load_glue(pk, d, st);
            } catch (const B2gError& e) { throw_error(e.code, "b2g_pk_group_load: key " + std::to_string(k) + ": " + e.what()); }
            glue[k] = {pk->d_tab_delta1, pk->d_tab_delta2, pk->d_tab_aa, pk->d_tab_bb};
            bidx_dev[k] = pk->d_bidx;
            consts_dev[k] = pk->d_consts;
        }
        g->d_keys = dev_upload<KeyGlue>(glue.data(), glue.size() * sizeof(KeyGlue), st);
        g->d_bidx = dev_upload<const uint32_t*>(bidx_dev.data(), bidx_dev.size() * sizeof(uint32_t*), st);
        g->d_consts = dev_upload<const uint8_t*>(consts_dev.data(), consts_dev.size() * sizeof(uint8_t*), st);
        CUDA_CHECK(cudaStreamSynchronize(st));
        guard.g = nullptr;
        *out = g;
    });
}

int b2g_pk_group_free(b2g_pk_group* g) {
    return guarded([&] {
        if (!g) return;
        DevGuard dg(g->device);
        cudaDeviceSynchronize();
        group_release(g);
    });
}

int b2g_prove_keys(b2g_ctx* ctx, b2g_pk_group* g, const uint32_t* counts, const void* r_canon, const void* s_canon, const void* const* w_mont,
                   uint8_t* proofs_out) {
    return guarded_clear([&] {
        if (!ctx || !g || !counts || !r_canon || !s_canon || !w_mont || !proofs_out) throw_error(B2G_E_SHAPE, "null pointer");
        if (ctx->shard_count != 1) throw_error(B2G_E_SHAPE, "b2g_prove_keys needs an unsharded context");
        ctx_idle(ctx);
        if (g->device != ctx->device) throw_error(B2G_E_SHAPE, "handle belongs to another device");
        const std::vector<KeyBases> bases = group_bases(g);
        GroupLayout L;
        for (int q = 0; q < NQ; q++) { L.c[q] = g->plan[q].c; L.row[q] = g->row[q]; }
        std::vector<uint32_t> n_vars, n_dom;
        for (size_t k = 0; k < g->keys.size(); k++) { n_vars.push_back(g->mats[k]->n_vars); n_dom.push_back(g->mats[k]->n); }
        const CallLayout C = call_layout(L, bases, n_vars, n_dom, counts);
        for (uint32_t j = 0; j < C.count; j++) if (!w_mont[j]) throw_error(B2G_E_SHAPE, "null witness " + std::to_string(j));
        DevGuard dg(ctx->device);
        const size_t table_bytes = C.rows.size() * sizeof(KeyedRow) + C.key_of.size() * 4;
        prove_pass(ctx, C.count, g->keys.size(), false, r_canon, s_canon, w_mont, n_vars.data(), C.key_of.data(),
                   [&] {
                       // every query holds count proofs of the mean base count of its sort (rounded up), at the group's window size
                       const int sb = g->b_sparse ? S_B : S_W;
                       const int sort_of[NQ] = {S_H, S_W, S_W, sb, sb};
                       uint32_t navg[NQ];
                       for (int q = 0; q < NQ; q++) navg[q] = std::max<uint32_t>(1, (uint32_t)((C.total_n[sort_of[q]] + C.count - 1) / C.count));
                       ensure_witness_buffers(ctx, C.total_w, C.total_v);
                       ensure_batch_buffers(ctx, C.count);
                       ensure_scratch(ctx, g->plan, navg, C.count, g->b_sparse, g->b_sparse ? C.total_n[S_B] : 0);
                       ensure_keyed_buffer(ctx, table_bytes);
                   },
                   [&] {
                       std::vector<uint8_t> table(table_bytes);
                       memcpy(table.data(), C.rows.data(), C.rows.size() * sizeof(KeyedRow));
                       memcpy(table.data() + C.rows.size() * sizeof(KeyedRow), C.key_of.data(), C.key_of.size() * 4);
                       CUDA_CHECK(cudaMemcpyAsync(ctx->d_keyed, table.data(), table_bytes, cudaMemcpyHostToDevice, ctx->st[0]));
                       std::vector<uint64_t> key = {g->uid, ctx->alloc_gen};
                       key.insert(key.end(), counts, counts + g->keys.size());
                       run_graph(ctx, ctx->graphs[G_KEYS], std::move(key), false, [&](bool) { enqueue_keys(ctx, g, C, counts); });
                   });
        CUDA_CHECK(cudaStreamSynchronize(ctx->st[0]));
        memcpy(proofs_out, ctx->h_proof, (size_t)C.count * 256);
    });
}

int b2g_pk_group_layout(uint32_t n_keys, const uint32_t* bases, const uint32_t* n_vars, const uint32_t* n_dom, const uint32_t* counts,
                        int32_t* c_out, uint32_t* row_out, uint64_t* rows_out) {
    return guarded([&] {
        if ((n_keys && !bases) || !c_out || !row_out || (counts && (!n_vars || !n_dom || !rows_out))) throw_error(B2G_E_SHAPE, "null pointer");
        std::vector<KeyBases> b(n_keys);
        for (uint32_t k = 0; k < n_keys; k++) for (int q = 0; q < NQ; q++) b[k][q] = bases[(size_t)k * NQ + q];
        const GroupLayout L = group_layout(b);
        for (int q = 0; q < NQ; q++) c_out[q] = L.c[q];
        for (uint32_t k = 0; k < n_keys; k++) for (int q = 0; q < NQ; q++) row_out[(size_t)k * NQ + q] = L.row[q][k];
        if (!counts) return;
        const CallLayout C = call_layout(L, b, std::vector<uint32_t>(n_vars, n_vars + n_keys), std::vector<uint32_t>(n_dom, n_dom + n_keys), counts);
        for (size_t i = 0; i < C.rows.size(); i++) {
            const KeyedRow& r = C.rows[i];
            rows_out[4 * i] = r.src; rows_out[4 * i + 1] = r.canon; rows_out[4 * i + 2] = r.n; rows_out[4 * i + 3] = r.row;
        }
    });
}

}  // extern "C"
