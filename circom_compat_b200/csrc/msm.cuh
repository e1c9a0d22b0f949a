// msm.cuh - multi-scalar multiplication sum_i k_i * P_i over BN254 G1 / G2 for a FIXED base set (a proving-key query).
//
// Replaces ark-ec 0.5.0 VariableBaseMSM::msm_bigint as called five times by ark-groth16 0.5.0
// create_proof_with_assignment (call sites /root/reference/src/zkey.rs:903-912, benches/groth16.rs:52-61; restated in
// SURVEY.md 3.4 / App. C.3).  Same signed base-2^c digit decomposition, but organised for H100:
//
//   * the bases never change between proofs, and HBM is 80 GB, so at key-load time every base P_i is expanded into the
//     affine table T[w][i] = 2^(c*w) * P_i (w = 0..nwin-1).  All windows then share ONE bucket set of 2^(c-1) buckets:
//     no per-window bucket reduction and no Horner doubling chain on the critical path.
//   * per proof: (1) canonical scalars + digit histogram (one thread per (window, scalar)), (2) exclusive scan,
//     (3) scatter of (table row | sign) into bucket-sorted order - a counting sort with warp-aggregated atomics, no
//     library sort; the sorted list is shared by every query that pairs the same scalars (L, A, B1, B2);
//     (4) perfectly load-balanced accumulation: each thread owns a fixed-length run of the sorted list, mixed-adds its
//     gathered bases in registers (XYZZ), and emits complete buckets directly and at most two boundary fragments;
//     (5) fragments are folded per bucket (big buckets by a whole CTA); (6) the weighted bucket sum sum_b (b+1)*B_b by
//     chunked running sums, a small double-and-add and a shared-memory tree.
//   Nothing in (1)-(6) synchronises with the host.
#pragma once
#include "ec.cuh"

namespace b2g {

constexpr int MSM_MAX_WIN = 32;          // c >= 8
constexpr int MSM_BIG_FRAGS = 32;        // buckets with more fragments than this are folded by a whole CTA

struct MsmPlan {                         // static per query
    uint32_t n = 0;                      // number of bases
    int c = 0, nwin = 0;
    uint32_t nbuckets = 0;               // 2^(c-1)
    void* table = nullptr;               // affine [nwin][n]
    bool g2 = false;
};

// Batched MSMs (b2g_prove_many): `count` scalar vectors against the same table are sorted into ONE list whose bucket key is
// j * nbuckets + b for proof j, so accumulation and fold run unchanged over count * nbuckets buckets.  Table rows, and so the
// entry word, do not depend on j.  The weighted reduction restarts its bucket weights per proof (grid.y = proof) and proof
// j's result is written at result + j * result_stride.
struct MsmScratch {                      // one per in-flight MSM
    uint32_t cap_n = 0; int cap_nwin = 0; uint32_t cap_buckets = 0; uint32_t chunk = 64; uint32_t sorted_n = 0; uint32_t reduce_chunk = 8;
    uint32_t cap_count = 1, sorted_count = 1;   // proofs the buffers hold / proofs in the last sort
    size_t result_stride = 0;                   // bytes between the results of consecutive proofs (0: one point)
    uint32_t *counts = nullptr, *offsets = nullptr, *cursor = nullptr, *entries = nullptr;
    uint32_t *big_list = nullptr, *big_count = nullptr;
    void *frag_first = nullptr, *frag_last = nullptr, *buckets = nullptr, *partials = nullptr, *result = nullptr;
    fe* scalars_canon = nullptr;         // n canonical scalars (filled by the digit pass)
    bool g2 = false, result_owned = false;
    cudaEvent_t prof0 = nullptr, prof1 = nullptr;   // optional: bracket the accumulate kernel (b2g_bench_msm)
    cudaStream_t tail = nullptr;                     // high-priority stream for the low-parallelism fold / weighted-sum kernels
    cudaEvent_t ev_acc = nullptr, ev_tail = nullptr;
};

// Window size by base count.  Larger windows than the textbook log2(n) - 3 pay off for small keys because the table removes
// the per-window reductions; from ~0.8 M bases up 15 windows of 17 bits beat 16 of 16 although the bucket set doubles
// (2^20 chain on one H100 80GB HBM3, 400 W power limit: 34.8 vs 33.4 proofs/s end to end).
// B2G_MSM_C overrides (8..22) for tuning.
inline int msm_pick_c(uint32_t n) {
    if (n >= 3u << 18) return 17;        // 15 windows instead of 16 pay for the doubled bucket set from ~0.8 M bases up
    if (n >= 1u << 19) return 16;
    if (n >= 1u << 15) return 15;
    if (n >= 1u << 13) return 13;
    if (n >= 1u << 11) return 11;
    int lg = 0; while ((1ull << (lg + 1)) <= n) lg++;
    return lg - 3 < 8 ? 8 : lg - 3;
}
inline int msm_nwin(int c) { return (255 + c - 1) / c; }

// Keyed batches (b2g_prove_keys): the proofs of one call belong to different keys whose tables of a query lie side by side
// in one arena built at one window size.  Proof j's row: its base count, its first scalar (elements into the scalar vector),
// its first slot of the canonical copy and the first arena row of its key (key k's row of base i in window w: row + w * n + i).
struct KeyedRow { uint64_t src; uint64_t canon; uint32_t n; uint32_t row; };
// sorts `count` proofs described by rows_dev (device) into one list of count * plan.nbuckets buckets; max_n / total_n: the
// largest and the summed n of the rows.  plan: the group's c, nwin, nbuckets and arena.
void msm_sort_keyed(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, bool scalars_mont, const KeyedRow* rows_dev, uint32_t count,
                    uint32_t max_n, uint64_t total_n, cudaStream_t st);
void msm_build_table_into(void* table, const void* bases_dev, uint32_t n, int c, bool g2, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ tableless streamed MSM
// sum_i rho^i P_i over bases read once (b2g_powers_msm, b2g_powers_check), in slices of at most POWERS_SLICE points.  No
// window table: a base costs one mixed addition per window, so every window keeps its own bucket set.  Per slice the scalars
// rho^(start + i) are made on the device (or given as a device vector: b2g_setup_check's transformed column weights), then
// the batched pipeline above runs with the window in the place of the proof:
// bucket key w * nbuckets + b, entry word = the base's index in the slice (| sign), accumulate and fold over the bases
// themselves, the weighted reduction restarting per window (grid.y) and giving one sum per window.  A Horner combine
// (c doublings per window) adds the slice's sum into a running device accumulator.
constexpr uint32_t POWERS_SLICE = 1u << 22;

// window size for n bases per slice: the least of nwin(c) * (n + 2^(c+1)) - one mixed addition per base and window, and the
// running-sum reduction's two additions per bucket - over c in [4, 20].  2^22 bases: c = 17 (15 windows).
inline int powers_pick_c(uint64_t n) {
    int best = 4;
    double cost = 1e300;
    for (int c = 4; c <= 20; c++) {
        const double k = (double)msm_nwin(c) * ((double)n + (double)(2ull << c));
        if (k < cost) { cost = k; best = c; }
    }
    return best;
}

struct PowersMsm {
    bool g2 = false;
    int c = 0, nwin = 0;
    uint32_t nbuckets = 0, cap = 0;     // buckets per window, bases per slice
    MsmScratch s;                       // counts / offsets / entries over nwin * nbuckets buckets, result = nwin window sums
    void* acc = nullptr;                // the running XYZZ sum
    fe* pw = nullptr;                   // rho^start, rho^POWERS_CHUNK (Montgomery)
};

// buffers for slices of up to `cap` bases; the window size is picked for `cap`
void powers_msm_alloc(PowersMsm& m, bool g2, uint32_t cap);
void powers_msm_free(PowersMsm& m);
// acc = infinity
void powers_msm_reset(PowersMsm& m, cudaStream_t st);
// acc += sum_{i < n} rho^(start + i) bases[i]: `bases` n affine Montgomery points on the device, `rho` one Montgomery Fr element
// on the device.  With `scalars` (n canonical Fr elements on the device) the slice takes them instead of the powers of rho, and
// rho and start are not read.  Nothing synchronises with the host.
void powers_msm_slice(PowersMsm& m, const void* bases, uint32_t n, uint64_t start, const fe* rho, cudaStream_t st,
                      const fe* scalars = nullptr);
// canon[i] = rho^(start + i) in canonical form, i < n (rho Montgomery, device); pw: 2 device Fr elements of scratch
void powers_scalars(const fe* rho, uint64_t start, uint32_t n, fe* pw, fe* canon, cudaStream_t st);

}  // namespace b2g
