// msm.cu - kernels and launchers of the fixed-base-table Pippenger MSM described in msm.cuh.
#include <type_traits>
#include "msm.cuh"
#include "util.cuh"

namespace b2g {

std::atomic<uint64_t> g_launch_count{0};

// ------------------------------------------------------------------------------------------------ key-load time
// T[w][i] = 2^(c*w) * P_i, affine.  One thread per base; the nwin XYZZ multiples live in local memory and are brought
// back to affine with one field inversion per thread (Montgomery's trick over ZZZ).
template <class C, class F>
__global__ void __launch_bounds__(128) msm_table_kernel(const void* __restrict__ bases, uint32_t n, int c, int nwin, void* __restrict__ table) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    using Pt = typename C::Pt; using Aff = typename C::Aff; using E = typename F::elem;
    Aff p = aff_load<F>(bases, i);
    if (C::aff_is_inf(p)) {
        Aff z; z.x = F::zero(); z.y = F::zero();
        for (int w = 0; w < nwin; w++) aff_store<F>(table, (size_t)w * n + i, z);
        return;
    }
    Pt pts[MSM_MAX_WIN];
    E pre[MSM_MAX_WIN];
    Pt cur = C::from_affine(p);
    E acc = F::one();
    for (int w = 0; w < nwin; w++) {
        pts[w] = cur;
        pre[w] = acc;
        acc = F::mul(acc, cur.zzz);                 // never zero: prime-order group, P != inf
        if (w + 1 < nwin) for (int j = 0; j < c; j++) cur = C::dbl(cur);
    }
    E inv = F::inv(acc);
    for (int w = nwin - 1; w >= 0; w--) {
        E iz = F::mul(inv, pre[w]);                 // 1/zzz_w
        inv = F::mul(inv, pts[w].zzz);
        Aff a;
        a.y = F::mul(pts[w].y, iz);
        a.x = F::mul(pts[w].x, F::mul(F::sqr(pts[w].zz), F::sqr(iz)));
        aff_store<F>(table, (size_t)w * n + i, a);
    }
}

// every base must be on the curve (or the all-zero point at infinity); *bad receives 1 + index of an offender
template <class C, class F>
__global__ void __launch_bounds__(256) msm_validate_kernel(const void* __restrict__ bases, uint32_t n, uint32_t* __restrict__ bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!aff_on_curve<C, F>(aff_load<F>(bases, i))) atomicMax(bad, i + 1u);
}

// ------------------------------------------------------------------------------------------------ (1) digits + histogram
// (1a) scalars -> canonical integers (one Montgomery reduction each).  (1a)-(1c) take proof j = blockIdx.y of a batch: its
// scalars start at j * scalar_stride, its canonical copy at j * n and its counters at j * nb.
__global__ void __launch_bounds__(256) msm_canon_kernel(const fe* __restrict__ scalars, uint32_t n, uint32_t scalar_stride, int scalars_mont, fe* __restrict__ canon_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    scalars += (size_t)blockIdx.y * scalar_stride;
    canon_out += (size_t)blockIdx.y * n;
    fe k = fe_load_nc(&scalars[i]);
    if (scalars_mont) k = Fr::to_canonical(k);
    fe_store(&canon_out[i], k);
}

// raw c-bit window w of a canonical scalar held in global memory
__device__ __forceinline__ uint32_t msm_window_bits(const uint32_t* __restrict__ k, int c, int w) {
    const uint32_t off = (uint32_t)w * (uint32_t)c, limb = off >> 5, sh = off & 31u;
    if (limb >= 8) return 0u;
    uint64_t v = __ldg(&k[limb]);
    if (limb + 1 < 8 && sh + (uint32_t)c > 32u) v |= (uint64_t)__ldg(&k[limb + 1]) << 32;
    return (uint32_t)(v >> sh) & ((1u << c) - 1u);
}

// Signed digit of window w without walking the whole carry chain (ark-ec make_digits semantics): the carry into window
// w is 1 iff the window below holds >= 2^(c-1), 0 iff it holds < 2^(c-1) - 1, and only for the single value
// 2^(c-1) - 1 does it depend on the next window down.
__device__ __forceinline__ int32_t msm_digit_at(const uint32_t* __restrict__ k, int c, int w) {
    const uint32_t half = 1u << (c - 1);
    uint32_t carry = 0;
    for (int v = w - 1; v >= 0; v--) {
        const uint32_t b = msm_window_bits(k, c, v);
        if (b >= half) { carry = 1; break; }
        if (b < half - 1) break;
    }
    const uint32_t coef = msm_window_bits(k, c, w) + carry;
    const uint32_t cout = (coef + half) >> c;
    return (int32_t)coef - (int32_t)(cout << c);
}

// (1b) one thread per (window, scalar): bucket histogram.  Hot buckets (circom witnesses: most wires are 0 / 1, so one bucket
// receives a large share of all entries) must not cost one atomic per entry, but match.any - the general way to group equal
// lanes - stalls the kernel on uniform scalars (profiled on the previous target GPU).  Two leader rounds do:
// the first pending lane broadcasts its bucket, every lane with the same bucket is counted by ONE atomic; a hot bucket is the
// leader's with high probability, and on uniform data the rounds cost four ballots.  Lanes still pending add individually.
constexpr int MSM_LEADER_ROUNDS = 2;

// histogram of the digits of one (window, scalar) pair per thread: `tid` < n * nwin of one proof's canonical scalars
__device__ __forceinline__ void msm_count_digits(const fe* __restrict__ canon, uint32_t n, int c, int nwin, uint32_t* __restrict__ counts, uint64_t tid) {
    const uint32_t w = (uint32_t)(tid / n), i = (uint32_t)(tid % n);
    int32_t d = 0;
    if (w < (uint32_t)nwin) d = msm_digit_at(canon[i].l, c, (int)w);
    const uint32_t b = d ? (uint32_t)(d < 0 ? -d : d) - 1u : 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31;
    bool pending = d != 0;
    {   // bucket 0 (digit +-1) is where the bits of a circom witness land: always grouped, one ballot
        const uint32_t hot = __ballot_sync(0xffffffffu, pending && b == 0u);
        if (hot) {
            if ((int)lane == __ffs(hot) - 1) atomicAdd(&counts[0], (uint32_t)__popc(hot));
            if (b == 0u) pending = false;
        }
    }
    #pragma unroll
    for (int round = 0; round < MSM_LEADER_ROUNDS; round++) {
        const uint32_t pend = __ballot_sync(0xffffffffu, pending);
        if (!pend) break;
        const int leader = __ffs(pend) - 1;
        const uint32_t lb = __shfl_sync(0xffffffffu, b, leader);
        const bool mine = pending && b == lb;
        const uint32_t same = __ballot_sync(0xffffffffu, mine);
        if ((int)lane == leader) atomicAdd(&counts[lb], (uint32_t)__popc(same));
        if (mine) pending = false;
    }
    if (pending) atomicAdd(&counts[b], 1u);
}

__global__ void __launch_bounds__(256) msm_count_kernel(const fe* __restrict__ canon, uint32_t n, int c, int nwin, uint32_t nb, uint32_t* __restrict__ counts) {
    canon += (size_t)blockIdx.y * n;
    counts += (size_t)blockIdx.y * nb;
    msm_count_digits(canon, n, c, nwin, counts, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}

// ------------------------------------------------------------------------------------------------ (2) exclusive scan (one CTA)
__global__ void __launch_bounds__(1024) msm_scan_kernel(const uint32_t* __restrict__ counts, uint32_t nb, uint32_t* __restrict__ offsets,
                                                        uint32_t* __restrict__ cursor) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry_s;
    const uint32_t tid = threadIdx.x, per = (nb + 1023u) / 1024u;
    const uint32_t lo = tid * per, hi = min(lo + per, nb);
    uint32_t s = 0;
    if ((per & 3u) == 0 && hi == lo + per) {                      // aligned chunk: independent 128-bit loads
        const uint4* v4 = reinterpret_cast<const uint4*>(counts + lo);
        #pragma unroll 4
        for (uint32_t j = 0; j < per / 4; j++) { const uint4 q = __ldg(&v4[j]); s += q.x + q.y + q.z + q.w; }
    } else {
        for (uint32_t j = lo; j < hi; j++) s += counts[j];
    }
    // block exclusive scan of s
    uint32_t v = s;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, v, d); if ((tid & 31) >= (uint32_t)d) v += t; }
    if ((tid & 31) == 31) warp_sums[tid >> 5] = v;
    __syncthreads();
    if (tid < 32) {
        uint32_t w = warp_sums[tid], x = w;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, x, d); if (tid >= (uint32_t)d) x += t; }
        warp_sums[tid] = x - w;
        if (tid == 31) carry_s = x;
    }
    __syncthreads();
    uint32_t run = warp_sums[tid >> 5] + v - s;
    for (uint32_t j = lo; j < hi; j++) { offsets[j] = run; cursor[j] = 0; run += counts[j]; }
    if (tid == 0) offsets[nb] = carry_s;
}

// ------------------------------------------------------------------------------------------------ (3) scatter
// the entries of one (window, scalar) pair per thread in bucket order: table row row0 + w * row_stride + i, bit 31 for a negative digit
__device__ __forceinline__ void msm_scatter_digits(const fe* __restrict__ canon, uint32_t n, uint32_t row0, uint32_t row_stride, int c, int nwin,
                                                   const uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor, uint32_t* __restrict__ entries,
                                                   uint64_t tid) {
    const uint32_t w = (uint32_t)(tid / n), i = (uint32_t)(tid % n);
    int32_t d = 0;
    if (w < (uint32_t)nwin) d = msm_digit_at(canon[i].l, c, (int)w);
    const uint32_t b = d ? (uint32_t)(d < 0 ? -d : d) - 1u : 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t entry = (row0 + w * row_stride + i) | (d < 0 ? 0x80000000u : 0u);
    bool pending = d != 0;
    {   // hot bucket 0 first (see msm_count_kernel)
        const uint32_t hot = __ballot_sync(0xffffffffu, pending && b == 0u);
        if (hot) {
            const int leader = __ffs(hot) - 1;
            uint32_t base = 0;
            if ((int)lane == leader) base = atomicAdd(&cursor[0], (uint32_t)__popc(hot));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (pending && b == 0u) {
                entries[offsets[0] + base + (uint32_t)__popc(hot & ((1u << lane) - 1u))] = entry;
                pending = false;
            }
        }
    }
    #pragma unroll
    for (int round = 0; round < MSM_LEADER_ROUNDS; round++) {            // same leader rounds as the histogram pass
        const uint32_t pend = __ballot_sync(0xffffffffu, pending);
        if (!pend) break;
        const int leader = __ffs(pend) - 1;
        const uint32_t lb = __shfl_sync(0xffffffffu, b, leader);
        const bool mine = pending && b == lb;
        const uint32_t same = __ballot_sync(0xffffffffu, mine);
        uint32_t base = 0;
        if ((int)lane == leader) base = atomicAdd(&cursor[lb], (uint32_t)__popc(same));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (mine) {
            entries[offsets[b] + base + (uint32_t)__popc(same & ((1u << lane) - 1u))] = entry;
            pending = false;
        }
    }
    if (pending) entries[offsets[b] + atomicAdd(&cursor[b], 1u)] = entry;
}

__global__ void __launch_bounds__(256) msm_scatter_kernel(const fe* __restrict__ canon, uint32_t n, uint32_t row_stride, int c, int nwin, uint32_t nb,
                                   const uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor, uint32_t* __restrict__ entries) {
    canon += (size_t)blockIdx.y * n;
    offsets += (size_t)blockIdx.y * nb;                    // global positions in the batch's one sorted list
    cursor += (size_t)blockIdx.y * nb;
    msm_scatter_digits(canon, n, 0u, row_stride, c, nwin, offsets, cursor, entries, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}

// ------------------------------------------------------------------------------------------------ (4) accumulate
// Run t = sorted positions [t*chunk, (t+1)*chunk), owned by one thread (G1) or one lane pair (G2).  Buckets that lie entirely
// inside the run are written to buckets[]; a run's first / last segment that belongs to a bucket crossing the run boundary
// goes to frag_first[t] / frag_last[t].

// slab_words != 0: the CTA's contiguous slab of the sorted entry list (128 runs = 32 KB at the default run length) is
// brought into shared memory by ONE bulk asynchronous copy (cp.async.bulk -> UBLKCP, completion on an mbarrier) instead of
// 64 strided 4-byte loads per run.  Every thread of the CTA calls this.
__device__ __forceinline__ void acc_stage_slab(uint32_t* slab, unsigned long long* slab_bar, const uint32_t* __restrict__ entries,
                                               uint64_t cta_first, uint32_t total, uint32_t slab_words) {
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(slab_bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0 && cta_first < total) {
        const uint64_t left = total - cta_first;
        const uint32_t bytes = (uint32_t)(((left < slab_words ? left : (uint64_t)slab_words) * 4 + 15) & ~15ull);    // the list is padded by 16 B
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"((uint32_t)__cvta_generic_to_shared(slab)), "l"(entries + cta_first), "r"(bytes), "r"(bar) : "memory");
    }
    if (cta_first < total) {
        uint32_t done = 0;
        while (!done)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar) : "memory");
    }
}

constexpr int MSM_SLAB_MAX_BYTES = 48 * 1024;   // larger G1 slabs are not staged: the runs read the entry list directly

// first bucket of the run starting at `start`: largest b with offsets[b] <= start, skipping empty buckets that share the offset
__device__ __forceinline__ uint32_t acc_first_bucket(const uint32_t* __restrict__ offsets, uint32_t nb, uint32_t start, uint32_t& bucket_end) {
    uint32_t lo = 0, hi = nb;                       // invariant: offsets[lo] <= start < offsets[hi]
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (offsets[mid] <= start) lo = mid; else hi = mid; }
    uint32_t b = lo;
    bucket_end = offsets[b + 1];
    while (bucket_end <= start) { b++; bucket_end = offsets[b + 1]; }
    return b;
}

// occupancy target: 4 CTAs/SM at 128 registers
template <class C, class F>
__global__ void __launch_bounds__(128, 4) msm_accumulate_kernel(const void* __restrict__ table, const uint32_t* __restrict__ entries,
                                      const uint32_t* __restrict__ offsets, uint32_t nb, uint32_t chunk,
                                      void* __restrict__ buckets, void* __restrict__ frag_first, void* __restrict__ frag_last, uint32_t slab_words) {
    using Pt = typename C::Pt; using Aff = typename C::Aff;
    const uint32_t total = offsets[nb];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t start64 = (uint64_t)t * chunk;
    extern __shared__ __align__(128) uint32_t slab[];
    __shared__ __align__(8) unsigned long long slab_bar;
    const uint64_t cta_first = (uint64_t)blockIdx.x * blockDim.x * chunk;
    if (slab_words) acc_stage_slab(slab, &slab_bar, entries, cta_first, total, slab_words);
    if (start64 >= total) return;
    const uint32_t start = (uint32_t)start64;
    const uint32_t end = (uint32_t)min((uint64_t)total, start64 + chunk);
    uint32_t bucket_end;
    uint32_t b = acc_first_bucket(offsets, nb, start, bucket_end);
    Pt acc = C::infinity();
    uint32_t seg_start = start;
    for (uint32_t pos = start; pos < end;) {
        // slab index pos - cta_first, formed in 32 bits: with the 64-bit cta_first live across the loop, CUDA 12.9 spills 8 B
        const uint32_t e = slab_words ? slab[pos - start + threadIdx.x * chunk] : entries[pos];
        Aff p = aff_load<F>(table, (size_t)(e & 0x7fffffffu));
        if (e >> 31) p.y = F::neg(p.y);
        C::madd(acc, p);
        pos++;
        if (pos == bucket_end || pos == end) {
            const uint32_t bucket_start = offsets[b];
            if (bucket_start >= start && bucket_end <= end) pt_store<F>(buckets, b, acc);
            else if (seg_start == start) pt_store<F>(frag_first, t, acc);
            else pt_store<F>(frag_last, t, acc);
            acc = C::infinity();
            seg_start = pos;
            if (pos == bucket_end && pos < end) {
                do { b++; bucket_end = offsets[b + 1]; } while (bucket_end <= pos);
            }
        }
    }
}

// G2: lane pair t (threads 2t, 2t+1 of the grid) owns run t and runs the lane-pair mixed addition of ec.cuh (G2Pair).  Both
// lanes walk the same entries; each loads its 64 B half of the 128 B table row (A: x, B: y - so the sign of an entry
// negates on lane B) and stores its two coordinates of the 256 B XYZZ record (A: X, ZZ at bytes 0 / 128; B: Y, ZZZ at 64 / 192).
// 3 CTAs x 128 threads per SM (166 registers, no stack): 192 chains per SM.  Capped at 128 registers for 4 CTAs/SM the kernel
// spills ~150 B per thread and measured slower (H100 80GB HBM3, 400 W: 9.04-9.08 ms vs 8.49-8.52 ms per 2^20 accumulation).
__global__ void __launch_bounds__(128, 3) msm_accumulate_g2_kernel(const void* __restrict__ table, const uint32_t* __restrict__ entries,
                                      const uint32_t* __restrict__ offsets, uint32_t nb, uint32_t chunk,
                                      void* __restrict__ buckets, void* __restrict__ frag_first, void* __restrict__ frag_last) {
    const uint32_t total = offsets[nb];
    const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 1;
    const uint32_t half = threadIdx.x & 1u;
    const bool A = half == 0;
    const unsigned mask = 3u << (threadIdx.x & 30u);
    const uint64_t start64 = (uint64_t)t * chunk;
    if (start64 >= total) return;
    const uint32_t start = (uint32_t)start64;
    const uint32_t end = (uint32_t)min((uint64_t)total, start64 + chunk);
    uint32_t bucket_end;
    uint32_t b = acc_first_bucket(offsets, nb, start, bucket_end);
    fe2 s0 = Fq2::zero(), s1 = Fq2::zero();
    bool empty = true;
    uint32_t seg_start = start;
    for (uint32_t pos = start; pos < end;) {
        const uint32_t e = entries[pos];
        fe2 qc;
        elem_load_nc(qc, (const char*)table + (size_t)(e & 0x7fffffffu) * 128 + half * 64);
        qc = Fq2::sel((e >> 31) && !A, Fq2::neg(qc), qc);
        G2Pair::madd(s0, s1, empty, qc, A, mask);
        pos++;
        if (pos == bucket_end || pos == end) {
            const uint32_t bucket_start = offsets[b];
            char* rec;
            if (bucket_start >= start && bucket_end <= end) rec = (char*)buckets + (size_t)b * 256;
            else if (seg_start == start) rec = (char*)frag_first + (size_t)t * 256;
            else rec = (char*)frag_last + (size_t)t * 256;
            elem_store(rec + half * 64, s0);
            elem_store(rec + 128 + half * 64, s1);
            s0 = Fq2::zero(); s1 = Fq2::zero(); empty = true;
            seg_start = pos;
            if (pos == bucket_end && pos < end) {
                do { b++; bucket_end = offsets[b + 1]; } while (bucket_end <= pos);
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------ (5) fold fragments
template <class C, class F>
__global__ void __launch_bounds__(128) msm_fold_kernel(const uint32_t* __restrict__ offsets, uint32_t nb, uint32_t chunk, void* __restrict__ buckets,
                                const void* __restrict__ frag_first, const void* __restrict__ frag_last,
                                uint32_t* __restrict__ big_list, uint32_t* __restrict__ big_count) {
    using Pt = typename C::Pt;
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    uint32_t s = offsets[b], e = offsets[b + 1];
    if (s == e) { pt_store<F>(buckets, b, C::infinity()); return; }
    uint32_t t0 = s / chunk, t1 = (e - 1) / chunk;
    if (t0 == t1) return;                                   // complete bucket, already written by (4)
    if (t1 - t0 + 1 > (uint32_t)MSM_BIG_FRAGS) { big_list[atomicAdd(big_count, 1u)] = b; return; }
    Pt acc = (s == t0 * chunk) ? pt_load<F>(frag_first, t0) : pt_load<F>(frag_last, t0);
    for (uint32_t t = t0 + 1; t <= t1; t++) { Pt q = pt_load<F>(frag_first, t); C::add(acc, q); }
    pt_store<F>(buckets, b, acc);
}

// sum of one point per thread; result valid in thread 0.  Inside a warp the partial sums travel by register shuffles
// (lane i adds lane i + d, d = 16 .. 1: the classic butterfly, every limb of the XYZZ point through __shfl_down_sync); the one
// or two warp results are then combined through shared memory.
template <class F> struct PtWords;
template <> struct PtWords<Fq> { static constexpr int N = 32; };
template <> struct PtWords<Fq2> { static constexpr int N = 64; };

template <class C, class F>
__device__ __forceinline__ typename C::Pt warp_sum_points(typename C::Pt v) {
    using Pt = typename C::Pt;
    static_assert(sizeof(Pt) == PtWords<F>::N * 4, "XYZZ point layout");
    #pragma unroll 1
    for (int d = 16; d > 0; d >>= 1) {
        Pt q;
        uint32_t* qw = reinterpret_cast<uint32_t*>(&q);
        const uint32_t* vw = reinterpret_cast<const uint32_t*>(&v);
        #pragma unroll
        for (int i = 0; i < PtWords<F>::N; i++) qw[i] = __shfl_down_sync(0xffffffffu, vw[i], d);
        if ((int)(threadIdx.x & 31) < d) C::add(v, q);
    }
    return v;
}

template <class C, class F, int NT>
__device__ __forceinline__ typename C::Pt block_sum_points(typename C::Pt v, typename C::Pt* sh) {
    static_assert(NT == 32 || NT == 64, "one or two warps");
    v = warp_sum_points<C, F>(v);
    if (NT == 32) return v;
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) { typename C::Pt q = sh[1]; C::add(v, q); }
    __syncthreads();                                       // sh may be reused by the caller's next round
    return v;
}

// Tail kernels (fold_big / reduce / sum) are latency chains on a few CTAs.  Their CTAs are kept smaller than one
// accumulation CTA (128 threads x 128 regs for G1) so that the block scheduler can slot them in as soon as a single
// accumulation CTA of a concurrently running query retires, instead of waiting for two slots on the same SM.
template <class F> struct TailThreads;
template <> struct TailThreads<Fq> { static constexpr int N = 64; };
template <> struct TailThreads<Fq2> { static constexpr int N = 32; };
constexpr int MSM_REDUCE_CHUNK_DEFAULT = 8;   // buckets per thread in the weighted reduction (B2G_MSM_REDUCE_CHUNK)

// buckets with many fragments: one CTA each
template <class C, class F>
__global__ void __launch_bounds__(TailThreads<F>::N) msm_fold_big_kernel(const uint32_t* __restrict__ offsets, uint32_t chunk, void* __restrict__ buckets,
                                    const void* __restrict__ frag_first, const void* __restrict__ frag_last,
                                    const uint32_t* __restrict__ big_list, const uint32_t* __restrict__ big_count) {
    using Pt = typename C::Pt;
    extern __shared__ __align__(32) unsigned char smem_raw[];
    Pt* sh = reinterpret_cast<Pt*>(smem_raw);
    const uint32_t nbig = *big_count;
    for (uint32_t bi = blockIdx.x; bi < nbig; bi += gridDim.x) {
        uint32_t b = big_list[bi];
        uint32_t s = offsets[b], e = offsets[b + 1];
        uint32_t t0 = s / chunk, t1 = (e - 1) / chunk;
        Pt acc = C::infinity();
        for (uint32_t t = t0 + threadIdx.x; t <= t1; t += TailThreads<F>::N) {
            Pt q = (t == t0 && s != t0 * chunk) ? pt_load<F>(frag_last, t0) : pt_load<F>(frag_first, t);
            C::add(acc, q);
        }
        Pt r = block_sum_points<C, F, TailThreads<F>::N>(acc, sh);
        if (threadIdx.x == 0) pt_store<F>(buckets, b, r);
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ (6) weighted bucket sum
// sum_b (b+1) * B_b.  Thread t takes buckets [t*S, (t+1)*S): running sums give A_t = sum_j (j+1) B_{tS+j} and
// S_t = sum_j B_{tS+j}; its contribution is A_t + (t*S) * S_t (small double-and-add); a CTA tree adds them up.
// blockIdx.y = proof of a batch: its nb buckets start at y * nb and its partials at y * gridDim.x, so the weights restart at 1.
template <class C, class F>
__global__ void __launch_bounds__(TailThreads<F>::N) msm_reduce_kernel(const void* __restrict__ buckets, uint32_t nb, uint32_t rchunk, void* __restrict__ partials) {
    using Pt = typename C::Pt;
    extern __shared__ __align__(32) unsigned char smem_raw[];
    Pt* sh = reinterpret_cast<Pt*>(smem_raw);
    buckets = (const char*)buckets + (size_t)blockIdx.y * nb * sizeof(Pt);
    partials = (char*)partials + (size_t)blockIdx.y * gridDim.x * sizeof(Pt);
    const uint32_t t = blockIdx.x * TailThreads<F>::N + threadIdx.x;
    const uint32_t base = t * rchunk;
    Pt run = C::infinity(), acc = C::infinity();
    if (base < nb) {
        const uint32_t cnt = min(rchunk, nb - base);
        for (int j = (int)cnt - 1; j >= 0; j--) {
            Pt q = pt_load<F>(buckets, base + j);
            C::add(run, q);
            C::add(acc, run);
        }
        // acc += base * run
        if (base != 0 && !C::is_inf(run)) {
            Pt m = C::infinity();
            int top = 31 - __clz(base);
            for (int i = top; i >= 0; i--) { m = C::dbl(m); if ((base >> i) & 1u) C::add(m, run); }
            C::add(acc, m);
        }
    }
    Pt r = block_sum_points<C, F, TailThreads<F>::N>(acc, sh);
    if (threadIdx.x == 0) pt_store<F>(partials, blockIdx.x, r);
}

// sum of `count` points (count <= a few hundred) by one CTA; CTA j sums points [j * count, (j + 1) * count) into out + j * out_stride
template <class C, class F>
__global__ void __launch_bounds__(TailThreads<F>::N) msm_sum_kernel(const void* __restrict__ pts, uint32_t count, void* __restrict__ out, size_t out_stride) {
    using Pt = typename C::Pt;
    extern __shared__ __align__(32) unsigned char smem_raw[];
    Pt* sh = reinterpret_cast<Pt*>(smem_raw);
    pts = (const char*)pts + (size_t)blockIdx.x * count * sizeof(Pt);
    out = (char*)out + (size_t)blockIdx.x * out_stride;
    Pt acc = C::infinity();
    for (uint32_t i = threadIdx.x; i < count; i += TailThreads<F>::N) { Pt q = pt_load<F>(pts, i); C::add(acc, q); }
    Pt r = block_sum_points<C, F, TailThreads<F>::N>(acc, sh);
    if (threadIdx.x == 0) pt_store<F>(out, 0, r);
}

// ------------------------------------------------------------------------------------------------ host side
static uint32_t env_u32(const char* name, uint32_t dflt) {
    const char* v = getenv(name);
    if (!v || !*v) return dflt;
    long x = strtol(v, nullptr, 10);
    return x > 0 ? (uint32_t)x : dflt;
}

// reference behaviour: an off-curve point in a zkey makes G1Affine::new / G2Affine::new panic (src/zkey.rs:340-360); here
// the load fails with B2G_E_INPUT.  `what` names the points in the message.
void msm_validate_points(const void* pts_dev, uint32_t n, bool g2, cudaStream_t st, const char* what) {
    if (n == 0) return;
    struct Flag { uint32_t* d = nullptr; ~Flag() { if (d) cudaFree(d); } } flag;
    uint32_t bad = 0;
    CUDA_CHECK(cudaMalloc(&flag.d, 4));
    CUDA_CHECK(cudaMemsetAsync(flag.d, 0, 4, st));
    if (g2) msm_validate_kernel<G2, Fq2><<<(n + 255) / 256, 256, 0, st>>>(pts_dev, n, flag.d);
    else msm_validate_kernel<G1, Fq><<<(n + 255) / 256, 256, 0, st>>>(pts_dev, n, flag.d);
    g_launch_count += 1;
    CUDA_CHECK(cudaMemcpyAsync(&bad, flag.d, 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    if (bad) throw_error(B2G_E_INPUT, std::string(g2 ? "G2" : "G1") + " point " + std::to_string(bad - 1) + " of " + what + " is not on the curve");
}

template <class C, class F>
static void msm_build_table_t(MsmPlan& plan, const void* bases_dev, uint32_t n, cudaStream_t st) {
    const size_t aff = 2 * Bytes<F>::ELEM;
    // B2G_MSM_C is a tuning override; outside [8, 22] the window count would overflow MSM_MAX_WIN or the bucket count 2^31
    uint32_t c = env_u32("B2G_MSM_C", (uint32_t)msm_pick_c(n ? n : 1));
    if (c < 8 || c > 22) throw_error(B2G_E_SHAPE, "B2G_MSM_C must be in [8, 22]");
    plan.n = n; plan.c = (int)c; plan.nwin = msm_nwin(plan.c); plan.nbuckets = 1u << (plan.c - 1);
    if (n == 0) { plan.table = nullptr; return; }
    if ((uint64_t)n * plan.nwin >= (1ull << 31)) throw_error(B2G_E_SHAPE, "msm: n * windows exceeds 2^31 table rows");
    msm_validate_points(bases_dev, n, plan.g2, st, "the query slice");
    CUDA_CHECK(cudaMalloc(&plan.table, (size_t)n * plan.nwin * aff));
    msm_table_kernel<C, F><<<(n + 127) / 128, 128, 0, st>>>(bases_dev, n, plan.c, plan.nwin, plan.table);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

void msm_build_table(MsmPlan& plan, const void* bases_dev, uint32_t n, bool g2, cudaStream_t st) {
    plan.g2 = g2;
    if (g2) msm_build_table_t<G2, Fq2>(plan, bases_dev, n, st);
    else msm_build_table_t<G1, Fq>(plan, bases_dev, n, st);
}

// rows [0, nwin(c) * n) of `table` (a key's place in a group's arena, b2g_pk_group_load) at a window size given by the group
void msm_build_table_into(void* table, const void* bases_dev, uint32_t n, int c, bool g2, cudaStream_t st) {
    if (n == 0) return;
    msm_validate_points(bases_dev, n, g2, st, "the query slice");
    if (g2) msm_table_kernel<G2, Fq2><<<(n + 127) / 128, 128, 0, st>>>(bases_dev, n, c, msm_nwin(c), table);
    else msm_table_kernel<G1, Fq><<<(n + 127) / 128, 128, 0, st>>>(bases_dev, n, c, msm_nwin(c), table);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

void msm_free_table(MsmPlan& plan) { if (plan.table) cudaFree(plan.table); plan.table = nullptr; }

// count: proofs of a batch the buffers hold (sorted entries, buckets, fragments and partials scale with it)
void msm_scratch_alloc(MsmScratch& s, uint32_t n, int nwin, uint32_t nbuckets_one, bool g2, bool with_sort, uint32_t count) {
    s.g2 = g2; s.cap_n = n; s.cap_nwin = nwin; s.cap_buckets = nbuckets_one; s.cap_count = count;
    s.chunk = env_u32(g2 ? "B2G_MSM_CHUNK_G2" : "B2G_MSM_CHUNK", env_u32("B2G_MSM_CHUNK", 64));
    const size_t pt = (g2 ? 4 * 64 : 4 * 32);
    const size_t nent = (size_t)n * nwin * count;
    const size_t nbuckets = (size_t)nbuckets_one * count;
    const size_t nchunks = (nent + s.chunk - 1) / s.chunk + 1;
    s.reduce_chunk = env_u32("B2G_MSM_REDUCE_CHUNK", MSM_REDUCE_CHUNK_DEFAULT);
    const size_t npart = ((size_t)nbuckets_one / (s.reduce_chunk * 32) + 64) * count;
    if (with_sort) {
        CUDA_CHECK(cudaMalloc(&s.counts, (size_t)nbuckets * 4));
        CUDA_CHECK(cudaMalloc(&s.offsets, ((size_t)nbuckets + 1) * 4));
        CUDA_CHECK(cudaMalloc(&s.cursor, (size_t)nbuckets * 4));
        CUDA_CHECK(cudaMalloc(&s.entries, (nent + 8) * 4));          // + 16 B: the bulk copy of the last slab is rounded up
        CUDA_CHECK(cudaMalloc(&s.scalars_canon, ((size_t)n * count + 1) * sizeof(fe)));
    }
    CUDA_CHECK(cudaMalloc(&s.big_list, (size_t)nbuckets * 4));
    CUDA_CHECK(cudaMalloc(&s.big_count, 4));
    CUDA_CHECK(cudaMalloc(&s.frag_first, nchunks * pt));
    CUDA_CHECK(cudaMalloc(&s.frag_last, nchunks * pt));
    CUDA_CHECK(cudaMalloc(&s.buckets, (size_t)nbuckets * pt));
    CUDA_CHECK(cudaMalloc(&s.partials, (npart + 1) * pt));
    CUDA_CHECK(cudaMalloc(&s.result, pt)); s.result_owned = true;
    // the tail kernels occupy a handful of CTAs for a long dependent chain: let them be dispatched ahead of the
    // thousands of pending accumulation CTAs of the other queries
    int least = 0, greatest = 0;
    CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    CUDA_CHECK(cudaStreamCreateWithPriority(&s.tail, cudaStreamNonBlocking, greatest));
    CUDA_CHECK(cudaEventCreateWithFlags(&s.ev_acc, cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&s.ev_tail, cudaEventDisableTiming));
}

void msm_scratch_free(MsmScratch& s) {
    void* ptrs[] = {s.counts, s.offsets, s.cursor, s.entries, s.big_list, s.big_count, s.frag_first, s.frag_last,
                    s.buckets, s.partials, s.result_owned ? s.result : nullptr, s.scalars_canon};
    for (void* p : ptrs) if (p) cudaFree(p);
    // a scratch that was never allocated, or whose allocation failed before the stream was made, has no tail stream
    if (s.tail) { cudaStreamDestroy(s.tail); cudaEventDestroy(s.ev_acc); cudaEventDestroy(s.ev_tail); }
    s = MsmScratch();
}

// count scalar vectors of n, the j-th at scalars_dev + j * scalar_stride, into one list of count * nbuckets buckets
void msm_sort(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, uint32_t n, bool scalars_mont, cudaStream_t st, uint32_t count,
              uint32_t scalar_stride) {
    if (n > plan.n) n = plan.n;                                  // msm_bigint truncates to the shorter side
    s.sorted_n = n; s.sorted_count = count;
    if (n == 0 || plan.table == nullptr) return;
    if (n > s.cap_n || plan.nwin > s.cap_nwin || plan.nbuckets > s.cap_buckets || count > s.cap_count || !s.entries) throw_error(B2G_E_SHAPE, "msm: sort scratch too small");
    const uint32_t nb = plan.nbuckets * count;
    constexpr unsigned SORT_CTA = 256;
    CUDA_CHECK(cudaMemsetAsync(s.counts, 0, (size_t)nb * 4, st));
    const dim3 pair_grid((unsigned)(((uint64_t)n * plan.nwin + SORT_CTA - 1) / SORT_CTA), count);
    msm_canon_kernel<<<dim3((n + SORT_CTA - 1) / SORT_CTA, count), SORT_CTA, 0, st>>>(scalars_dev, n, scalar_stride ? scalar_stride : n, scalars_mont ? 1 : 0, s.scalars_canon);
    msm_count_kernel<<<pair_grid, SORT_CTA, 0, st>>>(s.scalars_canon, n, plan.c, plan.nwin, plan.nbuckets, s.counts);
    msm_scan_kernel<<<1, 1024, 0, st>>>(s.counts, nb, s.offsets, s.cursor);
    // table rows are indexed w * plan.n + i (the table was built over plan.n bases, n may be shorter)
    msm_scatter_kernel<<<pair_grid, SORT_CTA, 0, st>>>(s.scalars_canon, n, plan.n, plan.c, plan.nwin, plan.nbuckets, s.offsets, s.cursor, s.entries);
    g_launch_count += 4;
    CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ keyed digit passes
// A batch whose proofs belong to different keys (b2g_prove_keys): proof j = blockIdx.y reads its own row of `rows` - base
// count n, first scalar, first canonical slot and the arena row of its key's table.  Its bucket key stays j * nb + b, so the
// scan, accumulation, fold and weighted reduction run unchanged.  A CTA past the proof's own n (or n * nwin) pairs leaves
// whole, so every warp that stays runs the ballots of the histogram and scatter with all its lanes.
__global__ void __launch_bounds__(256) msm_canon_keyed_kernel(const fe* __restrict__ scalars, const KeyedRow* __restrict__ rows, int scalars_mont,
                                                              fe* __restrict__ canon_out) {
    const KeyedRow r = rows[blockIdx.y];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    fe k = fe_load_nc(&scalars[r.src + i]);
    if (scalars_mont) k = Fr::to_canonical(k);
    fe_store(&canon_out[r.canon + i], k);
}

__global__ void __launch_bounds__(256) msm_count_keyed_kernel(const fe* __restrict__ canon, const KeyedRow* __restrict__ rows, int c, int nwin, uint32_t nb,
                                                              uint32_t* __restrict__ counts) {
    const KeyedRow r = rows[blockIdx.y];
    if ((uint64_t)blockIdx.x * blockDim.x >= (uint64_t)r.n * nwin) return;
    msm_count_digits(canon + r.canon, r.n, c, nwin, counts + (size_t)blockIdx.y * nb, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void __launch_bounds__(256) msm_scatter_keyed_kernel(const fe* __restrict__ canon, const KeyedRow* __restrict__ rows, int c, int nwin, uint32_t nb,
                                                                const uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor, uint32_t* __restrict__ entries) {
    const KeyedRow r = rows[blockIdx.y];
    if ((uint64_t)blockIdx.x * blockDim.x >= (uint64_t)r.n * nwin) return;
    msm_scatter_digits(canon + r.canon, r.n, r.row, r.n, c, nwin, offsets + (size_t)blockIdx.y * nb, cursor + (size_t)blockIdx.y * nb, entries,
                       (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}

void msm_sort_keyed(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, bool scalars_mont, const KeyedRow* rows_dev, uint32_t count,
                    uint32_t max_n, uint64_t total_n, cudaStream_t st) {
    // the accumulation sizes its runs by sorted_n * nwin * count: the mean base count per proof, rounded up, covers every entry
    s.sorted_n = (uint32_t)((total_n + count - 1) / count); s.sorted_count = count;
    if (total_n == 0 || plan.table == nullptr) { s.sorted_n = 0; return; }
    if (s.sorted_n > s.cap_n || plan.nwin > s.cap_nwin || plan.nbuckets > s.cap_buckets || count > s.cap_count || !s.entries)
        throw_error(B2G_E_SHAPE, "msm: keyed sort scratch too small");
    const uint32_t nb = plan.nbuckets * count;
    constexpr unsigned SORT_CTA = 256;
    CUDA_CHECK(cudaMemsetAsync(s.counts, 0, (size_t)nb * 4, st));
    const dim3 pair_grid((unsigned)(((uint64_t)max_n * plan.nwin + SORT_CTA - 1) / SORT_CTA), count);
    msm_canon_keyed_kernel<<<dim3((max_n + SORT_CTA - 1) / SORT_CTA, count), SORT_CTA, 0, st>>>(scalars_dev, rows_dev, scalars_mont ? 1 : 0, s.scalars_canon);
    msm_count_keyed_kernel<<<pair_grid, SORT_CTA, 0, st>>>(s.scalars_canon, rows_dev, plan.c, plan.nwin, plan.nbuckets, s.counts);
    msm_scan_kernel<<<1, 1024, 0, st>>>(s.counts, nb, s.offsets, s.cursor);
    msm_scatter_keyed_kernel<<<pair_grid, SORT_CTA, 0, st>>>(s.scalars_canon, rows_dev, plan.c, plan.nwin, plan.nbuckets, s.offsets, s.cursor, s.entries);
    g_launch_count += 4;
    CUDA_CHECK(cudaGetLastError());
}

// one accumulation launch over `nruns` runs: one thread per run for G1, one lane pair per run for G2 (64 runs per CTA)
template <class C, class F>
static void launch_accumulate(const void* table, const uint32_t* entries, const uint32_t* offsets, uint32_t nb, uint32_t chunk, uint32_t nruns,
                              const MsmScratch& s, cudaStream_t st) {
    constexpr bool g2 = std::is_same<F, Fq2>::value;
    constexpr uint32_t runs_per_cta = g2 ? 64u : 128u;
    const unsigned blocks = (unsigned)(((uint64_t)nruns + runs_per_cta - 1) / runs_per_cta);
    if constexpr (g2) {
        msm_accumulate_g2_kernel<<<blocks, 128, 0, st>>>(table, entries, offsets, nb, chunk, s.buckets, s.frag_first, s.frag_last);
    } else {
        const uint32_t slab_words = (size_t)chunk * runs_per_cta * 4 <= MSM_SLAB_MAX_BYTES ? chunk * runs_per_cta : 0u;
        msm_accumulate_kernel<C, F><<<blocks, 128, (size_t)slab_words * 4, st>>>(table, entries, offsets, nb, chunk, s.buckets, s.frag_first, s.frag_last, slab_words);
    }
}

template <class C, class F>
static void msm_accumulate_t(const MsmPlan& plan, const MsmScratch& sorted, MsmScratch& s, cudaStream_t st) {
    using Pt = typename C::Pt;
    const size_t ptb = sizeof(Pt);
    const uint32_t n = sorted.sorted_n, count = sorted.sorted_count;
    const size_t rstride = s.result_stride ? s.result_stride : ptb;
    if (n == 0 || plan.table == nullptr) { CUDA_CHECK(cudaMemset2DAsync(s.result, rstride, 0, ptb, count, st)); return; }
    if (plan.nbuckets > s.cap_buckets || n > s.cap_n || plan.nwin > s.cap_nwin || count > s.cap_count) throw_error(B2G_E_SHAPE, "msm: accumulate scratch too small");
    const uint32_t nb = plan.nbuckets * count, chunk = s.chunk;   // every proof's buckets in one range: runs cross proofs freely
    const uint32_t* offsets = sorted.offsets;
    CUDA_CHECK(cudaMemsetAsync(s.big_count, 0, 4, st));
    const uint64_t nent = (uint64_t)n * plan.nwin * count;
    const uint32_t nthreads = (uint32_t)((nent + chunk - 1) / chunk);
    if (s.prof0) CUDA_CHECK(cudaEventRecord(s.prof0, st));
    launch_accumulate<C, F>(plan.table, sorted.entries, offsets, nb, chunk, nthreads, s, st);
    if (s.prof1) CUDA_CHECK(cudaEventRecord(s.prof1, st));
    cudaStream_t main_st = st;
    CUDA_CHECK(cudaEventRecord(s.ev_acc, st)); CUDA_CHECK(cudaStreamWaitEvent(s.tail, s.ev_acc, 0)); st = s.tail;
    msm_fold_kernel<C, F><<<(nb + 127) / 128, 128, 0, st>>>(offsets, nb, chunk, s.buckets, s.frag_first, s.frag_last, s.big_list, s.big_count);
    constexpr int NT = TailThreads<F>::N;
    const size_t sh = (size_t)NT * ptb;
    msm_fold_big_kernel<C, F><<<128, NT, sh, st>>>(offsets, chunk, s.buckets, s.frag_first, s.frag_last, s.big_list, s.big_count);
    const uint32_t rchunk = s.reduce_chunk, nb1 = plan.nbuckets;
    const uint32_t nred = (nb1 + rchunk - 1) / rchunk;
    const uint32_t npart = (nred + NT - 1) / NT;                 // per proof
    msm_reduce_kernel<C, F><<<dim3(npart, count), NT, sh, st>>>(s.buckets, nb1, rchunk, s.partials);
    msm_sum_kernel<C, F><<<count, NT, sh, st>>>(s.partials, npart, s.result, rstride);
    CUDA_CHECK(cudaEventRecord(s.ev_tail, s.tail)); CUDA_CHECK(cudaStreamWaitEvent(main_st, s.ev_tail, 0));
    g_launch_count += 5;
    CUDA_CHECK(cudaGetLastError());
}

// bucket accumulation + reduction of `plan`'s table against an already sorted scalar vector (`sorted` may be shared by
// several queries that pair the same scalars with different bases: A, B1, B2, L all use the witness)
void msm_accumulate(const MsmPlan& plan, const MsmScratch& sorted, MsmScratch& acc, cudaStream_t st) {
    if (plan.g2) msm_accumulate_t<G2, Fq2>(plan, sorted, acc, st);
    else msm_accumulate_t<G1, Fq>(plan, sorted, acc, st);
}

void msm_run(const MsmPlan& plan, MsmScratch& s, const fe* scalars_dev, uint32_t n, bool scalars_mont, cudaStream_t st, uint32_t count,
             uint32_t scalar_stride) {
    msm_sort(plan, s, scalars_dev, n, scalars_mont, st, count, scalar_stride);
    msm_accumulate(plan, s, s, st);
}

// ------------------------------------------------------------------------------------------------ tableless streamed MSM
constexpr uint32_t POWERS_CHUNK = 16;            // consecutive powers one thread of powers_scalars_kernel makes

// pw[0] = rho^start, pw[1] = rho^POWERS_CHUNK (Montgomery), by square-and-multiply; one thread
__global__ void powers_base_kernel(const fe* __restrict__ rho, uint64_t start, fe* __restrict__ pw) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const fe r = *rho;
    fe acc = Fr::one(), sq = r;
    for (uint64_t e = start; e; e >>= 1) {
        if (e & 1) acc = Fr::mul(acc, sq);
        sq = Fr::sqr(sq);
    }
    pw[0] = acc;
    fe c = r;
    for (uint32_t k = 1; k < POWERS_CHUNK; k <<= 1) c = Fr::sqr(c);
    pw[1] = c;
}

// canon[i] = rho^(start + i) in canonical form, i < n: thread t starts from rho^start (rho^CHUNK)^t and multiplies by rho
__global__ void __launch_bounds__(256) powers_scalars_kernel(const fe* __restrict__ rho, const fe* __restrict__ pw, uint32_t n,
                                                             fe* __restrict__ canon) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i0 = t * POWERS_CHUNK;
    if (i0 >= n) return;
    fe x = pw[0], sq = pw[1];
    for (uint32_t e = t; e; e >>= 1) {
        if (e & 1) x = Fr::mul(x, sq);
        sq = Fr::sqr(sq);
    }
    const fe r = *rho;
    const uint32_t end = min(n, i0 + POWERS_CHUNK);
    for (uint32_t i = i0; i < end; i++) {
        fe_store(&canon[i], Fr::to_canonical(x));
        x = Fr::mul(x, r);
    }
}

// one thread per (window, scalar): the bucket key w * nb + |d| - 1 of every nonzero signed digit.  The scalars are powers of a
// random rho, so the digits are spread over the buckets and one atomic per entry does not contend.
__global__ void __launch_bounds__(256) powers_count_kernel(const fe* __restrict__ canon, uint32_t n, int c, int nwin, uint32_t nb,
                                                           uint32_t* __restrict__ counts) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t w = (uint32_t)(tid / n), i = (uint32_t)(tid % n);
    if (w >= (uint32_t)nwin) return;
    const int32_t d = msm_digit_at(canon[i].l, c, (int)w);
    if (d) atomicAdd(&counts[w * nb + (uint32_t)(d < 0 ? -d : d) - 1u], 1u);
}

// the entries in bucket order: the base's index in the slice, bit 31 for a negative digit
__global__ void __launch_bounds__(256) powers_scatter_kernel(const fe* __restrict__ canon, uint32_t n, int c, int nwin, uint32_t nb,
                                                             const uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor,
                                                             uint32_t* __restrict__ entries) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t w = (uint32_t)(tid / n), i = (uint32_t)(tid % n);
    if (w >= (uint32_t)nwin) return;
    const int32_t d = msm_digit_at(canon[i].l, c, (int)w);
    if (!d) return;
    const uint32_t key = w * nb + (uint32_t)(d < 0 ? -d : d) - 1u;
    entries[offsets[key] + atomicAdd(&cursor[key], 1u)] = i | (d < 0 ? 0x80000000u : 0u);
}

// acc += sum_w 2^(c w) W_w (Horner from the top window; one thread)
template <class C, class F>
__global__ void powers_horner_kernel(const void* __restrict__ windows, int nwin, int c, void* __restrict__ acc) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    typename C::Pt r = pt_load<F>(windows, nwin - 1);
    for (int w = nwin - 2; w >= 0; w--) {
        for (int k = 0; k < c; k++) r = C::dbl(r);
        C::add(r, pt_load<F>(windows, w));
    }
    typename C::Pt a = pt_load<F>(acc, 0);
    C::add(a, r);
    pt_store<F>(acc, 0, a);
}

void powers_msm_alloc(PowersMsm& m, bool g2, uint32_t cap) {
    m.g2 = g2;
    m.cap = cap ? cap : 1;
    m.c = powers_pick_c(m.cap);
    m.nwin = msm_nwin(m.c);
    m.nbuckets = 1u << (m.c - 1);
    const size_t pt = g2 ? 256 : 128, nb = (size_t)m.nbuckets * m.nwin;
    // the windows take the place of a batch's proofs: one "window" of nbuckets buckets per proof, nwin proofs
    msm_scratch_alloc(m.s, m.cap, 1, m.nbuckets, g2, false, (uint32_t)m.nwin);
    CUDA_CHECK(cudaMalloc(&m.s.counts, nb * 4));
    CUDA_CHECK(cudaMalloc(&m.s.offsets, (nb + 1) * 4));
    CUDA_CHECK(cudaMalloc(&m.s.cursor, nb * 4));
    CUDA_CHECK(cudaMalloc(&m.s.entries, ((size_t)m.cap * m.nwin + 8) * 4));    // + 16 B: the bulk copy of the last slab
    CUDA_CHECK(cudaMalloc(&m.s.scalars_canon, ((size_t)m.cap + POWERS_CHUNK) * sizeof(fe)));
    CUDA_CHECK(cudaFree(m.s.result));
    m.s.result = nullptr;
    CUDA_CHECK(cudaMalloc(&m.s.result, (size_t)m.nwin * pt));
    m.s.result_stride = pt;
    CUDA_CHECK(cudaMalloc(&m.acc, pt));
    CUDA_CHECK(cudaMalloc(&m.pw, 2 * sizeof(fe)));
}

void powers_msm_free(PowersMsm& m) {
    msm_scratch_free(m.s);
    if (m.acc) cudaFree(m.acc);
    if (m.pw) cudaFree(m.pw);
    m = PowersMsm();
}

void powers_msm_reset(PowersMsm& m, cudaStream_t st) { CUDA_CHECK(cudaMemsetAsync(m.acc, 0, m.g2 ? 256 : 128, st)); }

void powers_scalars(const fe* rho, uint64_t start, uint32_t n, fe* pw, fe* canon, cudaStream_t st) {
    if (n == 0) return;
    constexpr unsigned CTA = 256;
    powers_base_kernel<<<1, 1, 0, st>>>(rho, start, pw);
    powers_scalars_kernel<<<(n + POWERS_CHUNK * CTA - 1) / (POWERS_CHUNK * CTA), CTA, 0, st>>>(rho, pw, n, canon);
    g_launch_count += 2;
    CUDA_CHECK(cudaGetLastError());
}

template <class C, class F>
static void powers_msm_slice_t(PowersMsm& m, const void* bases, uint32_t n, uint64_t start, const fe* rho, cudaStream_t st,
                               const fe* scalars) {
    if (n == 0) return;
    if (n > m.cap) throw_error(B2G_E_SHAPE, "powers msm: slice larger than its buffers");
    constexpr unsigned CTA = 256;
    const uint32_t nb = m.nbuckets * (uint32_t)m.nwin;
    if (!scalars) {
        powers_scalars(rho, start, n, m.pw, m.s.scalars_canon, st);
        scalars = m.s.scalars_canon;
    }
    CUDA_CHECK(cudaMemsetAsync(m.s.counts, 0, (size_t)nb * 4, st));
    const unsigned blocks = (unsigned)(((uint64_t)n * m.nwin + CTA - 1) / CTA);
    powers_count_kernel<<<blocks, CTA, 0, st>>>(scalars, n, m.c, m.nwin, m.nbuckets, m.s.counts);
    msm_scan_kernel<<<1, 1024, 0, st>>>(m.s.counts, nb, m.s.offsets, m.s.cursor);
    powers_scatter_kernel<<<blocks, CTA, 0, st>>>(scalars, n, m.c, m.nwin, m.nbuckets, m.s.offsets, m.s.cursor, m.s.entries);
    g_launch_count += 3;
    CUDA_CHECK(cudaGetLastError());
    MsmPlan plan;
    plan.n = n; plan.c = m.c; plan.nwin = 1; plan.nbuckets = m.nbuckets; plan.table = const_cast<void*>(bases); plan.g2 = m.g2;
    m.s.sorted_n = n; m.s.sorted_count = (uint32_t)m.nwin;
    msm_accumulate_t<C, F>(plan, m.s, m.s, st);
    powers_horner_kernel<C, F><<<1, 1, 0, st>>>(m.s.result, m.nwin, m.c, m.acc);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

void powers_msm_slice(PowersMsm& m, const void* bases, uint32_t n, uint64_t start, const fe* rho, cudaStream_t st, const fe* scalars) {
    if (m.g2) powers_msm_slice_t<G2, Fq2>(m, bases, n, start, rho, st, scalars);
    else powers_msm_slice_t<G1, Fq>(m, bases, n, start, rho, st, scalars);
}

// A full entry slab is 48 KiB (128 runs x 96 entries) on top of the G1 accumulation kernel's static mbarrier word, which is
// more than the default dynamic limit (48 KiB minus the static size): without the opt-in such launches fail with "invalid
// argument".  The tail kernels use < 48 KiB of dynamic shared memory.
void msm_init_kernels() {
    CUDA_CHECK(cudaFuncSetAttribute(msm_accumulate_kernel<G1, Fq>, cudaFuncAttributeMaxDynamicSharedMemorySize, MSM_SLAB_MAX_BYTES));
}

}  // namespace b2g
