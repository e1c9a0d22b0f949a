// verify.cu - Groth16 verification of many proofs in one device pass (b2g_vk_load / b2g_vk_free / b2g_verify_many).
//
// Device counterpart of the host verifier the reference's users call right after proving (GrothBn::process_vk +
// verify_with_processed_vk, /root/reference/src/zkey.rs:868-870, 914-916; ark-groth16 0.5.0): a proof (A, B, C) with public
// inputs x is valid iff
//     e(A, B) * e(IC[0] + sum_i x_i IC[i + 1], -gamma) * e(C, -delta) == e(alpha, beta).
// The key is prepared once on the device (b2g_vk_load, or b2g_vk_load_many for many keys in the same four launches): on-curve
// checks, e(alpha, beta), the line coefficients of the two fixed G2 arguments -gamma and -delta for every loop step (ark's
// G2Prepared), and an 8-bit window table per IC[i + 1].
// A batch then runs four kernels, one proof per thread (the parallelism comes from the batch):
//   inputs   one warp per (proof, input): x_i IC[i + 1] from the window table (32 look-ups and a warp tree)
//   prepare  parse the proof (canonical coordinates; >= p or off the curve -> invalid), sum the prepared inputs, affine
//   miller   one multi-Miller loop over (A, B), (prepared, -gamma), (C, -delta) sharing one f; only B is stepped here
//   final    the final exponentiation, compared with e(alpha, beta) -> one verdict byte
// b2g_verify_batch, b2g_verify_batch_locate and b2g_verify_batch_keys check a random linear combination instead (weights r_i
// from the caller), once per segment of consecutive proofs under one key:
//     prod e(r_i A_i, B_i) * e(sum r_i C_i, -delta) * e(s_0 IC[0] + sum_j s_j IC[j], -gamma) == e(alpha, beta)^s_0,
//     s_0 = sum r_i, s_j = sum r_i x_ij (mod r), x_ij the j-th public input of proof i (j = 1..n_public), sums over the segment
// b2g_verify_batch runs it with one segment of the whole batch; b2g_verify_batch_locate with segments of LOCATE_GROUP proofs
// whose sums leave out the malformed proofs (a mask), then b2g_verify_many on the well-formed proofs of the segments that
// fail; b2g_verify_batch_keys with one segment per key; b2g_verify_batch_keys_locate with segments of LOCATE_GROUP proofs of
// one key, then one b2g_verify_many pass whose kernels check each proof under its own key.  A segment table and a table of
// key records drive every stage below.
//   prepare  one proof per thread: the parse and on-curve checks above, r_i A_i (affine) and r_i C_i (XYZZ)
//   g2       one proof per thread: the proof parses and its B lies in G2 (the mask)
//   scalars  one CTA per (chunk of at most SCALAR_CHUNK proofs of a segment, j): partial sums of r_i x_ij (x_i0 = 1)
//   inputs   one warp per (segment, j): s_j from the segment's partial sums, then s_j IC[j] from the key's window table
//            (IC[0]: a variable-base product)
//   miller   one proof per thread: the one-pair Miller loop of (r_i A_i, B_i)
//   reduce   per segment: the product of the Miller values and the sums of the r_i C_i and of the s_j IC[j], in levels of
//            one CTA per at most 64 or 128 records of one segment, until each segment has one value
//   pairs    one segment per thread: the Miller loop of the two prepared pairs
//   rhs      one segment per thread: e(alpha, beta)^s_0
//   final    one segment per thread: one final exponentiation, compared with rhs -> one verdict byte per segment
// Only prepare -> miller -> product -> final run on the context's stream; the rest runs next to them on two side streams.
// b2g_proofs_decompress and the _compressed verifiers take arkworks' 128-byte compressed proofs: a decode kernel (one proof
// per thread) writes the 256-byte rows the kernels above read, and a second kernel checks that each decoded B lies in G2 (the
// batch check leaves that to batch_g2_kernel).  The decoding rules are restated above decompress_kernel.
// b2g_rerandomize_many (ark-groth16's rerandomize_proof) parses rows with the verifiers' proof_parse and runs one kernel, one
// proof per thread: rerandomize_kernel.
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>
#include "../../include/b2groth.h"
#include "fixed.cuh"
#include "pairing.cuh"
#include "stage.cuh"
#include "util.cuh"
#include "verify.cuh"

using namespace b2g;

constexpr uint32_t TABLE_POINTS = 32 * 255;         // entries of one 8-bit window table
constexpr size_t TABLE_BYTES = TABLE_POINTS * 64;    // one 8-bit window table of a G1 point
constexpr size_t F12_BYTES = 384;

// the device memory of one b2g_vk_load_many call: every key's arrays, carved out of one allocation.  Each handle the call
// made holds a reference; the last one to be freed frees the allocation.
struct VkArena {
    uint8_t* base = nullptr;
    ~VkArena() { if (base) cudaFree(base); }
};

struct b2g_vk {
    int device = 0;
    uint32_t n_public = 0;
    std::shared_ptr<VkArena> arena;   // the memory the arrays below lie in
    uint8_t* d_g1 = nullptr;       // alpha, IC[0..n_public] (G1 affine, Montgomery, 64 B each)
    uint8_t* d_g2 = nullptr;       // beta, gamma, delta (G2 affine, 128 B each)
    uint8_t* d_lines = nullptr;    // prepared lines of -gamma, then of -delta: 2 x ATE_LINES x LINE_BYTES
    uint8_t* d_eab = nullptr;      // e(alpha, beta), 384 B
    uint8_t* d_tabs = nullptr;     // window tables of IC[1..n_public], TABLE_BYTES apart (none when n_public == 0)
    bool gamma_inf = false, delta_inf = false;
};

namespace b2g {

// Per-proof record written by the prepare kernel: A (64 B), B (128 B), C (64 B), the prepared inputs (64 B), all affine
// Montgomery, then a word that is 1 when the proof's points parsed and lie on their curves.
constexpr size_t REC_BYTES_V = 384, REC_OK = 320;

struct VerifyBufs {
    size_t cap_count = 0, cap_pub = 0, cap_part = 0, cap_batch = 0, cap_comp = 0, cap_meta = 0;
    uint8_t *d_proofs = nullptr, *d_rec = nullptr, *d_f = nullptr, *d_verdict = nullptr;   // per proof
    uint8_t *d_pub = nullptr, *d_part = nullptr;                                            // per (proof, input)
    uint8_t* d_batch = nullptr;                   // the batch check's scratch: weights, reduction levels, group tails, ...
    uint8_t* d_comp = nullptr;                    // compressed proofs (128 B each), then one decoded-ok byte per proof
    uint8_t* d_meta = nullptr;                    // b2g_verify_many's key records and segment table
    cudaStream_t side[2] = {nullptr, nullptr};    // the batch check's tail pieces, next to the per-proof kernels
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    std::vector<uint8_t> h_meta;                  // the key records, segment table and reduction spans of the last call (host)
};

void verify_bufs_free(VerifyBufs* v) {
    if (!v) return;
    for (cudaStream_t s : v->side) if (s) cudaStreamDestroy(s);
    for (cudaEvent_t e : v->ev) if (e) cudaEventDestroy(e);
    for (void* p : {(void*)v->d_proofs, (void*)v->d_rec, (void*)v->d_f, (void*)v->d_verdict, (void*)v->d_pub, (void*)v->d_part,
                    (void*)v->d_batch, (void*)v->d_comp, (void*)v->d_meta}) if (p) cudaFree(p);
    delete v;
}

// ------------------------------------------------------------------------------------------------ key and segment tables
// the key a segment is checked under: its prepared lines of -gamma and -delta, e(alpha, beta), the window tables of
// IC[1..n_public], alpha and IC (b2g_vk's arrays), and whether each prepared pair takes part (gamma, delta not at infinity)
struct KeyRec {
    const uint8_t *lines, *eab, *tabs, *g1;
    uint32_t n_public, gamma_on, delta_on, pad;
};
// a segment: proofs first .. first + count - 1 under key record `key`; its public inputs start at scalar `pub`.  In the batch
// check, its (chunk, j) work items of batch_scalars_kernel start at `part` (chunks of them, chunk-major: chunk q's item j is
// part + q * (n_public + 1) + j) and its prepared-input points at `pt`; b2g_verify_many's kernels leave those three at 0.
// first, pub, part and pt never decrease along the table.
struct Seg {
    uint64_t pub;
    uint32_t key, first, count, part, chunks, pt;
};

// one key of a b2g_vk_load_many call as its kernels read it: where its arrays lie in the call's allocation, its first point
// of vk_validate_kernel and its first window table of vk_tables_kernel (pt and tab never decrease along the table)
struct VkRec {
    uint64_t pt, tab;
    uint8_t *g1, *g2, *eab, *lines, *tabs;
    uint32_t n_public, pad;
};

// the last record k < n with s[k].*M <= v, for a field that is nondecreasing along the table (a Seg's first, part, pt, or the
// 64-bit pub; a VkRec's pt or tab)
template <auto M, class R, class T>
__device__ __forceinline__ uint32_t seg_find(const R* __restrict__ s, uint32_t n, T v) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s[mid].*M <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// ------------------------------------------------------------------------------------------------ kernels
// b2g_verify_many's kernels check each proof under its own key: proof j belongs to the segment whose first .. first + count -
// 1 holds it, and its public inputs (and their G1 records in part) start at seg.pub + (j - seg.first) * n_public.  A call
// under one key is a table of one segment.
// x * IC[i + 1] for one (proof, input) per warp: w indexes the public-input scalars of every proof back to back, input i of
// proof j of the segment whose inputs hold w; pub = canonical scalars, part = G1 XYZZ records (both w-indexed)
__global__ void __launch_bounds__(128) verify_inputs_kernel(const KeyRec* __restrict__ keys, const Seg* __restrict__ segs, uint32_t n_segs,
                                                            const uint32_t* __restrict__ pub, size_t total, uint8_t* __restrict__ part) {
    __shared__ G1::Pt sh[4][32];
    const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= total) return;                                // whole warps leave together
    // a segment without inputs shares its pub with the next one, so the last segment with pub <= w is the one that holds w
    const Seg s = segs[seg_find<&Seg::pub>(segs, n_segs, (uint64_t)w)];
    const KeyRec& key = keys[s.key];
    const uint32_t i = (uint32_t)((w - s.pub) % key.n_public);
    G1::Pt p = warp_fixed_mul<G1, Fq>(key.tabs + (size_t)i * TABLE_BYTES, pub + 8 * w, sh[threadIdx.x >> 5]);
    if ((threadIdx.x & 31) == 0) pt_store<Fq>(part, w, p);
}

// a canonical coordinate below p
__device__ __forceinline__ bool fe_below_p(const fe& a) {
    const uint32_t p[8] = {FqParams::P0, FqParams::P1, FqParams::P2, FqParams::P3, FqParams::P4, FqParams::P5, FqParams::P6, FqParams::P7};
    for (int i = 7; i >= 0; i--) if (a.l[i] != p[i]) return a.l[i] < p[i];
    return false;
}

// a 256-byte proof as affine Montgomery points; true when every coordinate is below p and every point on its curve
__device__ __forceinline__ bool proof_parse(const uint8_t* pr, G1::Aff& a, G2::Aff& b, G1::Aff& cc) {
    fe c[8];
    bool ok = true;
    for (int k = 0; k < 8; k++) { const fe v = fe_load(pr + 32 * k); ok &= fe_below_p(v); c[k] = Fq::from_canonical(v); }
    a.x = c[0]; a.y = c[1]; b.x.c0 = c[2]; b.x.c1 = c[3]; b.y.c0 = c[4]; b.y.c1 = c[5]; cc.x = c[6]; cc.y = c[7];
    return ok && aff_on_curve<G1, Fq>(a) && aff_on_curve<G1, Fq>(cc) && aff_on_curve<G2, Fq2>(b);
}

__global__ void __launch_bounds__(128) verify_prepare_kernel(const uint8_t* __restrict__ proofs, const KeyRec* __restrict__ keys,
                                                             const Seg* __restrict__ segs, uint32_t n_segs, const uint8_t* __restrict__ part,
                                                             uint32_t count, uint8_t* __restrict__ rec) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    G1::Aff a, cc; G2::Aff b;
    const bool ok = proof_parse(proofs + (size_t)j * 256, a, b, cc);
    const Seg s = segs[seg_find<&Seg::first>(segs, n_segs, j)];
    const KeyRec& key = keys[s.key];
    const uint32_t n_public = key.n_public;
    const size_t p0 = s.pub + (size_t)(j - s.first) * n_public;
    G1::Pt acc = G1::from_affine(aff_load<Fq>(key.g1, 1));   // IC[0]
    for (uint32_t i = 0; i < n_public; i++) G1::add(acc, pt_load<Fq>(part, p0 + i));
    uint8_t* r = rec + (size_t)j * REC_BYTES_V;
    aff_store<Fq>(r, 0, a);
    aff_store<Fq2>(r + 64, 0, b);
    aff_store<Fq>(r + 192, 0, cc);
    aff_store<Fq>(r + 256, 0, G1::to_affine(acc));
    *reinterpret_cast<uint32_t*>(r + REC_OK) = ok;
}

__global__ void __launch_bounds__(64) verify_miller_kernel(const uint8_t* __restrict__ rec, const KeyRec* __restrict__ keys,
                                                           const Seg* __restrict__ segs, uint32_t n_segs, uint32_t count,
                                                           uint8_t* __restrict__ fout) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const uint8_t* r = rec + (size_t)j * REC_BYTES_V;
    if (!*reinterpret_cast<const uint32_t*>(r + REC_OK)) return;
    const KeyRec& key = keys[segs[seg_find<&Seg::first>(segs, n_segs, j)].key];
    const uint8_t* lines = key.lines;
    const G1::Aff a = aff_load<Fq>(r, 0), c = aff_load<Fq>(r + 192, 0), prep = aff_load<Fq>(r + 256, 0);
    const G2::Aff b = aff_load<Fq2>(r + 64, 0);
    G1::Aff fp[2];
    const uint8_t* fl[2];
    int nfix = 0;
    if (key.gamma_on && !G1::aff_is_inf(prep)) { fp[nfix] = prep; fl[nfix++] = lines; }
    if (key.delta_on && !G1::aff_is_inf(c)) { fp[nfix] = c; fl[nfix++] = lines + ATE_LINES * LINE_BYTES; }
    fe12 f;
    miller_loop(f, !G1::aff_is_inf(a) && !G2::aff_is_inf(b), a, b, nfix, fp, fl);
    Fq12::store(fout + (size_t)j * F12_BYTES, f);
}

__global__ void __launch_bounds__(64) verify_final_kernel(const uint8_t* __restrict__ rec, const uint8_t* __restrict__ fin,
                                                          const KeyRec* __restrict__ keys, const Seg* __restrict__ segs, uint32_t n_segs,
                                                          uint32_t count, uint8_t* __restrict__ verdict) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    if (!*reinterpret_cast<const uint32_t*>(rec + (size_t)j * REC_BYTES_V + REC_OK)) { verdict[j] = 0; return; }
    fe12 e;
    Fq12::final_exponentiation(e, Fq12::load(fin + (size_t)j * F12_BYTES));
    verdict[j] = Fq12::eq(e, Fq12::load(keys[segs[seg_find<&Seg::first>(segs, n_segs, j)].key].eab));
}

// ---------------------------------------------------------------------------------------------- batch check kernels
// b2g_verify_batch, b2g_verify_batch_locate and b2g_verify_batch_keys: the batch equation once per segment of consecutive
// proofs under one key, each segment's products and sums optionally masked by wf (wf[i] = 1 when proof i parses and its B
// lies in G2).
// Per-proof record, REC_BYTES_V apart: r A (affine, 64 B), B (affine, 128 B), r C (XYZZ, 128 B).  The record area is zeroed
// first, so a proof that does not parse keeps r A and r C at infinity.  The ok word starts all ones and any failed parse,
// on-curve or G2 check clears it.
constexpr size_t BREC_B = 64, BREC_RC = 192;
// tail values of a segment, segment g's at tails + g * TAIL_BYTES (Fq12 384 B, G1 XYZZ 128 B): the product of the per-proof
// Miller values, the Miller value of the prepared pairs, e(alpha, beta)^s_0, sum r C, the prepared inputs, s_0
constexpr size_t TAIL_F = 0, TAIL_G = 384, TAIL_RHS = 768, TAIL_RC = 1152, TAIL_PREP = 1280, TAIL_S0 = 1408, TAIL_BYTES = 1536;
static_assert(TAIL_BYTES % 256 == 0, "segment tails stay 256-byte aligned");
constexpr uint32_t LOCATE_GROUP = 64;              // proofs per segment of b2g_verify_batch_locate: one CTA of f12_product_kernel
constexpr uint32_t SCALAR_CHUNK = 2048;            // at most this many proofs per CTA of batch_scalars_kernel

// one CTA of a segmented reduction: records first .. first + n - 1 of one segment, to value `out` of the next level, or to
// the tail of segment out & ~TO_TAIL when TO_TAIL is set
struct Span { uint32_t first, n, out; };
constexpr uint32_t TO_TAIL = 0x80000000u;

__device__ __forceinline__ uint8_t* span_out(const Span& s, uint8_t* dst, size_t rec_bytes, uint8_t* tails) {
    return s.out & TO_TAIL ? tails + (size_t)(s.out & ~TO_TAIL) * TAIL_BYTES : dst + (size_t)s.out * rec_bytes;
}

__device__ __forceinline__ void weight_load(uint32_t* k, const uint32_t* w, size_t i) {
    for (int t = 0; t < 4; t++) k[t] = w[4 * i + t];
}

__global__ void __launch_bounds__(128) batch_prepare_kernel(const uint8_t* __restrict__ proofs, const uint32_t* __restrict__ w,
                                                            uint32_t count, uint8_t* __restrict__ rec, uint32_t* __restrict__ ok_all) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    G1::Aff a, cc; G2::Aff b;
    // a failed proof's record is not written: it stays zeroed, so its r A and r C are at infinity, and the cleared ok word
    // fails a batch verdict (a group verdict leaves the proof out through wf instead)
    if (!proof_parse(proofs + (size_t)j * 256, a, b, cc)) { atomicAnd(ok_all, 0u); return; }
    uint32_t k[4];
    weight_load(k, w, j);
    uint8_t* r = rec + (size_t)j * REC_BYTES_V;
    aff_store<Fq>(r, 0, G1::to_affine(G1::mul_affine(a, k, 4)));
    aff_store<Fq2>(r + BREC_B, 0, b);
    pt_store<Fq>(r + BREC_RC, 0, G1::mul_affine(cc, k, 4));
}

// one proof per thread, on a side stream next to the per-proof chain: wf[j] = the proof parses and its B lies in G2; clears
// the ok word when it does not
__global__ void __launch_bounds__(128) batch_g2_kernel(const uint8_t* __restrict__ proofs, uint32_t count, uint8_t* __restrict__ wf,
                                                       uint32_t* __restrict__ ok_all) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    G1::Aff a, cc; G2::Aff b;
    const bool good = proof_parse(proofs + (size_t)j * 256, a, b, cc) && g2_in_subgroup(b);
    wf[j] = good;
    if (!good) atomicAnd(ok_all, 0u);
}

// CTA t, the work item (chunk q of segment s, j): part[t] = the sum over the proofs i of the chunk (SCALAR_CHUNK proofs
// from s.first + q * SCALAR_CHUNK, fewer at the segment's end) of r_i (j = 0) or of Fr::mul(r_i, x_ij) = r_i x_ij / R
// (j >= 1), leaving out proof i when mask[i] = 0 (no mask: every proof)
__global__ void __launch_bounds__(128) batch_scalars_kernel(const uint32_t* __restrict__ w, const uint32_t* __restrict__ pub,
                                                            const uint8_t* __restrict__ mask, const Seg* __restrict__ segs,
                                                            uint32_t n_segs, const KeyRec* __restrict__ keys, uint8_t* __restrict__ part) {
    __shared__ fe sh[128];
    const Seg s = segs[seg_find<&Seg::part>(segs, n_segs, blockIdx.x)];
    const uint32_t n_public = keys[s.key].n_public, q = (blockIdx.x - s.part) / (n_public + 1), j = (blockIdx.x - s.part) % (n_public + 1);
    const uint32_t end = s.first + min(s.count, (q + 1) * SCALAR_CHUNK);
    fe acc = Fr::zero();
    for (uint32_t i = s.first + q * SCALAR_CHUNK + threadIdx.x; i < end; i += 128) {
        if (mask && !mask[i]) continue;
        fe wi = fe_zero();
        weight_load(wi.l, w, i);
        acc = Fr::add(acc, j ? Fr::mul(wi, fe_load(pub + 8 * (s.pub + (size_t)(i - s.first) * n_public + j - 1))) : wi);
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int d = 64; d > 0; d >>= 1) {
        if ((int)threadIdx.x < d) sh[threadIdx.x] = Fr::add(sh[threadIdx.x], sh[threadIdx.x + d]);
        __syncthreads();
    }
    if (threadIdx.x == 0) fe_store(part + (size_t)blockIdx.x * 32, sh[0]);
}

// one warp per prepared-input point t < n_pts_all, point j = t - seg.pt of segment g (j = 0..n_public of its key): s_gj = the
// sum of the segment's chunk sums of batch_scalars_kernel, then pts[t] = s_gj IC[j] (IC[0]: a variable-base product); s_g0
// to the segment's tail
__global__ void __launch_bounds__(128) batch_inputs_kernel(const uint8_t* __restrict__ part, const Seg* __restrict__ segs, uint32_t n_segs,
                                                           const KeyRec* __restrict__ keys, uint32_t n_pts_all,
                                                           uint8_t* __restrict__ pts, uint8_t* __restrict__ tails) {
    __shared__ G1::Pt sh[4][32];
    __shared__ fe s[4];
    const uint32_t wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t t = (size_t)blockIdx.x * 4 + wid;
    if (t >= n_pts_all) return;                            // whole warps leave together
    const uint32_t g = seg_find<&Seg::pt>(segs, n_segs, (uint32_t)t);
    const Seg sg = segs[g];
    const KeyRec& key = keys[sg.key];
    const uint32_t n_pts = key.n_public + 1, j = (uint32_t)t - sg.pt;
    const uint8_t *tabs = key.tabs, *g1 = key.g1;
    fe acc = Fr::zero();
    for (uint32_t q = lane; q < sg.chunks; q += 32) acc = Fr::add(acc, fe_load(part + ((size_t)sg.part + (size_t)q * n_pts + j) * 32));
    for (int d = 16; d > 0; d >>= 1) {
        fe o;
        for (int q = 0; q < 8; q++) o.l[q] = __shfl_down_sync(0xffffffffu, acc.l[q], d);
        acc = Fr::add(acc, o);
    }
    if (lane == 0) s[wid] = j ? Fr::from_canonical(acc) : acc;   // from_canonical cancels the products' 1 / R
    __syncwarp();
    if (j) {
        const G1::Pt p = warp_fixed_mul<G1, Fq>(tabs + (size_t)(j - 1) * TABLE_BYTES, s[wid].l, sh[wid]);
        if (lane == 0) pt_store<Fq>(pts, t, p);
    } else if (lane == 0) {
        pt_store<Fq>(pts, t, G1::mul_scalar(G1::from_affine(aff_load<Fq>(g1, 1)), s[wid].l));
        fe_store(tails + (size_t)g * TAIL_BYTES + TAIL_S0, s[wid]);
    }
}

__global__ void __launch_bounds__(64) batch_miller_kernel(const uint8_t* __restrict__ rec, const uint32_t* __restrict__ ok_all,
                                                          uint32_t count, uint8_t* __restrict__ fout) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    fe12 f = Fq12::one();
    if (*ok_all) {
        const uint8_t* r = rec + (size_t)j * REC_BYTES_V;
        const G1::Aff a = aff_load<Fq>(r, 0);
        const G2::Aff b = aff_load<Fq2>(r + BREC_B, 0);
        if (!G1::aff_is_inf(a) && !G2::aff_is_inf(b)) miller_loop_t<true, 0>(f, a, b, nullptr, nullptr);
    }
    Fq12::store(fout + (size_t)j * F12_BYTES, f);
}

// CTA b, span sp = spans[b] (n <= 64): the product of src[sp.first .. sp.first + sp.n - 1] (Fq12, `stride` bytes apart),
// taking 1 for record i when mask[i] = 0 (no mask: every record), to dst (F12_BYTES apart) or to a tail (at tails)
__global__ void __launch_bounds__(64) f12_product_kernel(const uint8_t* __restrict__ src, size_t stride, const Span* __restrict__ spans,
                                                         const uint8_t* __restrict__ mask, uint8_t* __restrict__ dst, uint8_t* __restrict__ tails) {
    __shared__ fe12 sh[64];
    const Span sp = spans[blockIdx.x];
    const uint32_t t = threadIdx.x, i = sp.first + t;
    sh[t] = t < sp.n && (!mask || mask[i]) ? Fq12::load(src + (size_t)i * stride) : Fq12::one();
    __syncthreads();
    for (uint32_t d = 32; d > 0; d >>= 1) {
        if (t < d) { fe12 x = sh[t]; Fq12::mul(x, x, sh[t + d]); sh[t] = x; }
        __syncthreads();
    }
    if (t == 0) Fq12::store(span_out(sp, dst, F12_BYTES, tails), sh[0]);
}

// CTA b, span sp = spans[b]: the sum of src[sp.first .. sp.first + sp.n - 1] (G1 XYZZ, `stride` bytes apart), leaving out
// record i when mask[i] = 0 (no mask: every record), to dst (128 B apart) or to a tail (at tails)
__global__ void __launch_bounds__(128) g1_sum_kernel(const uint8_t* __restrict__ src, size_t stride, const Span* __restrict__ spans,
                                                     const uint8_t* __restrict__ mask, uint8_t* __restrict__ dst, uint8_t* __restrict__ tails) {
    __shared__ G1::Pt sh[128];
    const Span sp = spans[blockIdx.x];
    const uint32_t t = threadIdx.x, end = sp.first + sp.n;
    sh[t] = G1::infinity();                                // accumulated in shared memory: a register sum spills
    for (uint32_t i = sp.first + t; i < end; i += 128)
        if (!mask || mask[i]) { G1::Pt x = sh[t]; G1::add(x, pt_load<Fq>(src + (size_t)i * stride, 0)); sh[t] = x; }
    __syncthreads();
    for (uint32_t d = 64; d > 0; d >>= 1) {
        if (t < d) { G1::Pt x = sh[t]; G1::add(x, sh[t + d]); sh[t] = x; }
        __syncthreads();
    }
    if (t == 0) pt_store<Fq>(span_out(sp, dst, 128, tails), 0, sh[0]);
}

// the Miller value of the prepared pairs (prepared inputs, -gamma) and (sum r C, -delta); 1 when both drop out
__device__ __forceinline__ void tail_pairs(uint8_t* tail, const uint8_t* lines, bool gamma_on, bool delta_on) {
    const G1::Aff prep = G1::to_affine(pt_load<Fq>(tail + TAIL_PREP, 0)), c = G1::to_affine(pt_load<Fq>(tail + TAIL_RC, 0));
    G1::Aff fp[2];
    const uint8_t* fl[2];
    int nfix = 0;
    if (gamma_on && !G1::aff_is_inf(prep)) { fp[nfix] = prep; fl[nfix++] = lines; }
    if (delta_on && !G1::aff_is_inf(c)) { fp[nfix] = c; fl[nfix++] = lines + ATE_LINES * LINE_BYTES; }
    G2::Aff none; none.x = Fq2::zero(); none.y = Fq2::zero();
    fe12 g;
    miller_loop(g, false, fp[0], none, nfix, fp, fl);
    Fq12::store(tail + TAIL_G, g);
}

// one segment per thread: the Miller value of the segment's prepared pairs, with the lines of the segment's key
__global__ void __launch_bounds__(64) batch_pairs_kernel(uint8_t* __restrict__ tails, uint32_t n_segs, const Seg* __restrict__ segs,
                                                         const KeyRec* __restrict__ keys) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_segs) return;
    const KeyRec& key = keys[segs[g].key];
    tail_pairs(tails + (size_t)g * TAIL_BYTES, key.lines, key.gamma_on, key.delta_on);
}

// one segment per thread: e(alpha, beta)^s_g0 of the segment's key
__global__ void __launch_bounds__(64) batch_rhs_kernel(uint8_t* __restrict__ tails, uint32_t n_segs, const Seg* __restrict__ segs,
                                                       const KeyRec* __restrict__ keys) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_segs) return;
    uint8_t* tail = tails + (size_t)g * TAIL_BYTES;
    fe12 rhs;
    const fe s0 = fe_load(tail + TAIL_S0);
    Fq12::cyclotomic_exp(rhs, Fq12::load(keys[segs[g].key].eab), s0.l);
    Fq12::store(tail + TAIL_RHS, rhs);
}

// the final exponentiation of (per-proof product) x (prepared pairs) equals e(alpha, beta)^s_0
__device__ __forceinline__ bool tail_holds(const uint8_t* tail) {
    fe12 f = Fq12::load(tail + TAIL_F), e;
    Fq12::mul(f, f, Fq12::load(tail + TAIL_G));
    Fq12::final_exponentiation(e, f);
    return Fq12::eq(e, Fq12::load(tail + TAIL_RHS));
}

// one segment per thread: verdict[g] = the ok word is set (no ok word: always), the segment's ok byte is set (no ok bytes:
// always) and the segment's batch equation holds.  A segment whose proofs are all masked out has every value at 1 (product,
// pairs and e(alpha, beta)^0), so it holds.
__global__ void __launch_bounds__(64) batch_final_kernel(const uint8_t* __restrict__ tails, uint32_t n_segs, const uint32_t* __restrict__ ok_all,
                                                         const uint8_t* __restrict__ seg_ok, uint8_t* __restrict__ verdict) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < n_segs) verdict[g] = (!ok_all || *ok_all) && (!seg_ok || seg_ok[g]) && tail_holds(tails + (size_t)g * TAIL_BYTES);
}

// one proof per thread, after batch_g2_kernel: clears the ok byte of the segment that holds a proof with wf[j] = 0, so that
// a malformed proof fails its own segment only (b2g_verify_batch_keys)
__global__ void __launch_bounds__(128) batch_segment_ok_kernel(const uint8_t* __restrict__ wf, const Seg* __restrict__ segs, uint32_t n_segs,
                                                               uint32_t count, uint8_t* __restrict__ seg_ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < count && !wf[j]) seg_ok[seg_find<&Seg::first>(segs, n_segs, j)] = 0;
}

// b2g_test_op ops 43-45: G2 membership of a G2 affine point (out: 8 B, 1 or 0), r * P for a G1 affine P and a 128-bit r
// (b: 16 B; out: 64 B affine), f^k for a cyclotomic Fq12 f and a canonical 256-bit k (b: 32 B; out: 384 B)
__global__ void batch_test_kernel(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (op == 43) {
        const uint64_t v = g2_in_subgroup(aff_load<Fq2>(a, i));
        reinterpret_cast<uint64_t*>(out)[i] = v;
    } else if (op == 44) {
        uint32_t k[4];
        weight_load(k, reinterpret_cast<const uint32_t*>(b), i);
        aff_store<Fq>(out, i, G1::to_affine(G1::mul_affine(aff_load<Fq>(a, i), k, 4)));
    } else {
        fe12 r;
        const fe k = fe_load(b + (size_t)i * 32);
        Fq12::cyclotomic_exp(r, Fq12::load(a + (size_t)i * F12_BYTES), k.l);
        Fq12::store(out + (size_t)i * F12_BYTES, r);
    }
}

// ---------------------------------------------------------------------------------------------- compressed proofs
// Proof::<Bn254>::deserialize_compressed (ark-serialize, ark-ec and ark-ff 0.5, Validate::Yes), restated:
//   layout    A = bytes 0-31, B = bytes 32-95, C = bytes 96-127, little-endian.  A G1 point is x; a G2 point is x.c0 (no
//             flags) followed by x.c1.  The flags are the top two bits of the point's last byte (of x, or of x.c1).
//   flags     bit 7: y is the larger of {y, -y}; bit 6: infinity; both set: invalid (SWFlags::from_u8 gives None)
//   range     with the flags masked off, every Fq value (x, x.c0, x.c1) is below p, even when the infinity flag is set
//   infinity  the point is infinity and x is otherwise ignored; decoded as all-zero coordinates, as b2g_prove writes it
//   otherwise y^2 = x^3 + 3 (G1) or x^3 + 3 / (9 + u) (G2) must have a square root; of the two roots, the smaller one when
//             bit 7 is clear and the larger one when it is set, in the order of canonical values (Fq2: c1 first, then c0)
//   subgroup  B is in G2 (G1 has cofactor 1: A and C need no check)
// An undecodable proof becomes a row of 0xFF bytes: every coordinate is then >= p, so proof_parse refuses it and both
// verifiers report it invalid with their kernels unchanged.
constexpr size_t COMP_BYTES = 128;

// the coordinate that carries a point's flags: its value with the flags cleared, flags = bit 7 << 1 | bit 6
__device__ __forceinline__ fe comp_load(const uint8_t* p, uint32_t& flags) {
    fe x = fe_load(p);
    flags = x.l[7] >> 30;
    x.l[7] &= 0x3fffffffu;
    return x;
}

// canonical a > b
__device__ __forceinline__ bool fe_greater(const fe& a, const fe& b) {
    for (int i = 7; i >= 0; i--) if (a.l[i] != b.l[i]) return a.l[i] > b.l[i];
    return false;
}
// a canonical y is the larger of {y, -y} (Fq::neg is the same modular subtraction on canonical values)
__device__ __forceinline__ bool y_is_larger(const fe& y) { return fe_greater(y, Fq::neg(y)); }
__device__ __forceinline__ bool y_is_larger(const fe2& y) {
    const fe n1 = Fq::neg(y.c1);
    return fe_equal(y.c1, n1) ? fe_greater(y.c0, Fq::neg(y.c0)) : fe_greater(y.c1, n1);
}
__device__ __forceinline__ fe to_canon(const fe& a) { return Fq::to_canonical(a); }
__device__ __forceinline__ fe2 to_canon(const fe2& a) { fe2 r; r.c0 = Fq::to_canonical(a.c0); r.c1 = Fq::to_canonical(a.c1); return r; }
__device__ __forceinline__ fe to_mont(const fe& a) { return Fq::from_canonical(a); }
__device__ __forceinline__ fe2 to_mont(const fe2& a) { fe2 r; r.c0 = Fq::from_canonical(a.c0); r.c1 = Fq::from_canonical(a.c1); return r; }
__device__ __forceinline__ bool field_sqrt(fe& r, const fe& a) { bool ok; r = Fq::sqrt(a, ok); return ok; }
__device__ __forceinline__ bool field_sqrt(fe2& r, const fe2& a) { return Fq2::sqrt(r, a); }

// the canonical y of the point with canonical x on y^2 = x^3 + b, the root the sign flag picks; false when there is none
template <class F>
__device__ __forceinline__ bool decompress_y(typename F::elem& y, const typename F::elem& x, bool larger) {
    const typename F::elem xm = to_mont(x);
    typename F::elem r;
    if (!field_sqrt(r, F::add(F::mul(F::sqr(xm), xm), curve_b((const F*)nullptr)))) return false;
    y = to_canon(r);
    if (y_is_larger(y) != larger) y = F::neg(y);
    return true;
}

// a compressed G1 point (32 B) -> canonical x, y (zeros at infinity); false when it does not decode
__device__ __forceinline__ bool g1_decompress(fe* out, const uint8_t* p) {
    uint32_t f;
    const fe x = comp_load(p, f);
    if (f == 3 || !fe_below_p(x)) return false;
    if (f & 1) { out[0] = fe_zero(); out[1] = fe_zero(); return true; }
    out[0] = x;
    return decompress_y<Fq>(out[1], x, f & 2);
}

// a compressed G2 point (64 B) -> canonical x.c0, x.c1, y.c0, y.c1 (zeros at infinity), without the subgroup check
__device__ __forceinline__ bool g2_decompress(fe* out, const uint8_t* p) {
    uint32_t f;
    fe2 x, y;
    x.c0 = fe_load(p);
    x.c1 = comp_load(p + 32, f);
    if (f == 3 || !fe_below_p(x.c0) || !fe_below_p(x.c1)) return false;
    if (f & 1) { for (int k = 0; k < 4; k++) out[k] = fe_zero(); return true; }
    if (!decompress_y<Fq2>(y, x, f & 2)) return false;
    out[0] = x.c0; out[1] = x.c1; out[2] = y.c0; out[3] = y.c1;
    return true;
}

// k canonical coordinates, or k x 32 bytes of 0xFF when !ok
__device__ __forceinline__ void coords_store(uint8_t* p, const fe* c, int k, bool ok) {
    fe ff;
    for (int i = 0; i < 8; i++) ff.l[i] = 0xffffffffu;
    for (int i = 0; i < k; i++) fe_store(p + 32 * i, ok ? c[i] : ff);
}

// one proof per thread: compressed row j -> the canonical 256-byte row j of b2g_prove and ok[j] = 1, or the 0xFF row and
// ok[j] = 0.  No subgroup check: decompress_g2_kernel adds it where the caller needs it.
__global__ void __launch_bounds__(128) decompress_kernel(const uint8_t* __restrict__ comp, uint32_t count, uint8_t* __restrict__ proofs,
                                                         uint8_t* __restrict__ ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const uint8_t* in = comp + (size_t)j * COMP_BYTES;
    fe c[8];
    for (int k = 0; k < 8; k++) c[k] = fe_zero();
    const bool good = g1_decompress(c, in) && g2_decompress(c + 2, in + 32) && g1_decompress(c + 6, in + 96);
    coords_store(proofs + (size_t)j * 256, c, 8, good);
    ok[j] = good;
}

// G2 membership of every decoded B, one proof per thread, in its own kernel so that the decoder does not carry
// g2_in_subgroup's registers and stack: a row whose B is outside G2 becomes the 0xFF row and ok[j] = 0
__global__ void __launch_bounds__(128) decompress_g2_kernel(uint32_t count, uint8_t* __restrict__ proofs, uint8_t* __restrict__ ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count || !ok[j]) return;
    uint8_t* row = proofs + (size_t)j * 256;
    G2::Aff b;
    b.x.c0 = to_mont(fe_load(row + 64)); b.x.c1 = to_mont(fe_load(row + 96));
    b.y.c0 = to_mont(fe_load(row + 128)); b.y.c1 = to_mont(fe_load(row + 160));
    if (!g2_in_subgroup(b)) { coords_store(row, nullptr, 8, false); ok[j] = 0; }
}

// b2g_test_op ops 46-48: the Fq square root (a: 32 B Montgomery; out: 64 B), the Fq2 square root (a: 64 B; out: 96 B), and
// one compressed G2 point decoded without the subgroup check (a: 64 B; out: 160 B: the canonical affine point, or 0xFF
// bytes).  Each result is followed by a 32-byte slot whose first word is 1 when there is a root / the point decodes.
__global__ void decompress_test_kernel(int op, const uint8_t* __restrict__ a, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool ok;
    uint8_t* o;
    if (op == 46) {
        o = out + (size_t)i * 64;
        fe_store(o, Fq::sqrt(fe_load(a + (size_t)i * 32), ok));
        o += 32;
    } else if (op == 47) {
        o = out + (size_t)i * 96;
        fe2 x, r;
        elem_load(x, a + (size_t)i * 64);
        ok = Fq2::sqrt(r, x);
        elem_store(o, r);
        o += 64;
    } else {
        o = out + (size_t)i * 160;
        fe c[4];
        for (int k = 0; k < 4; k++) c[k] = fe_zero();
        ok = g2_decompress(c, a + (size_t)i * 64);
        coords_store(o, c, 4, ok);
        o += 128;
    }
    fe flag = fe_zero();
    flag.l[0] = ok;
    fe_store(o, flag);
}

// ---------------------------------------------------------------------------------------------- key points
// b2g_points_serialize / b2g_points_deserialize: CanonicalSerialize / CanonicalDeserialize (Validate::Yes) of bare G1 or G2
// affine points, the elements of a serialized ProvingKey<Bn254> or VerifyingKey<Bn254> (ark-groth16 0.5).  The compressed
// form and its rules are those above COMP_BYTES.  The uncompressed form is x then y (G2: x.c0, x.c1, y.c0, y.c1) with the
// point's flags on the last byte of y (of y.c1): bit 7 is written for the larger y and ignored on read, bit 6 = infinity
// (zero coordinates on write), both set is invalid.  On read, every coordinate with the flags masked off must be below p,
// even under the infinity flag; a point without the infinity flag must lie on its curve; a G2 point not at infinity must lie
// in G2, in both forms (points_g2_subgroup_kernel).  One point per thread, in slices of at most KEY_SLICE points.
constexpr size_t KEY_SLICE = size_t(1) << 20;

__device__ __forceinline__ void as_elem(fe& r, const fe* c) { r = c[0]; }
__device__ __forceinline__ void as_elem(fe2& r, const fe* c) { r.c0 = c[0]; r.c1 = c[1]; }

// one point per thread: Montgomery point i (all zero = infinity) -> its canonical bytes with flags; a coordinate >= p lowers
// *bad to base + i
template <class F>
__global__ void __launch_bounds__(128) points_serialize_kernel(const uint8_t* __restrict__ pts, uint32_t n, int compress, uint64_t base,
                                                               uint8_t* __restrict__ out, unsigned long long* __restrict__ bad) {
    constexpr int K = Bytes<F>::ELEM / 32;                 // Fq coordinates of one of x, y
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe c[2 * K];
    bool ok = true, inf = true;
    for (int k = 0; k < 2 * K; k++) {
        c[k] = fe_load(pts + ((size_t)i * 2 * K + k) * 32);
        ok &= fe_below_p(c[k]);
        inf &= fe_equal(c[k], fe_zero());
        c[k] = to_canon(c[k]);
    }
    if (!ok) { atomicMin(bad, (unsigned long long)(base + i)); return; }
    typename F::elem y;
    as_elem(y, c + K);
    const int last = compress ? K - 1 : 2 * K - 1;         // the coordinate that carries the flags
    c[last].l[7] |= inf ? 0x40000000u : (y_is_larger(y) ? 0x80000000u : 0u);
    uint8_t* o = out + (size_t)i * (last + 1) * 32;
    for (int k = 0; k <= last; k++) fe_store(o + 32 * k, c[k]);
}

// one point per thread: serialized point i -> Montgomery point i (all zero = infinity), or zeros and *bad lowered to base + i
// when it does not decode.  No subgroup check: points_g2_subgroup_kernel adds it for G2.
template <class C, class F, bool COMPRESS>
__global__ void __launch_bounds__(128) points_deserialize_kernel(const uint8_t* __restrict__ in, uint32_t n, uint64_t base,
                                                                 uint8_t* __restrict__ pts, unsigned long long* __restrict__ bad) {
    constexpr int K = Bytes<F>::ELEM / 32;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe c[2 * K];
    for (int k = 0; k < 2 * K; k++) c[k] = fe_zero();
    const uint8_t* p = in + (size_t)i * (COMPRESS ? K : 2 * K) * 32;
    bool ok;
    if constexpr (COMPRESS) {
        if constexpr (K == 1) ok = g1_decompress(c, p); else ok = g2_decompress(c, p);
        for (int k = 0; k < 2 * K; k++) c[k] = to_mont(c[k]);
    } else {
        uint32_t f;
        for (int k = 0; k < 2 * K - 1; k++) c[k] = fe_load(p + 32 * k);
        c[2 * K - 1] = comp_load(p + 32 * (2 * K - 1), f);
        ok = f != 3;
        for (int k = 0; k < 2 * K; k++) ok &= fe_below_p(c[k]);
        if (ok && (f & 1)) {
            for (int k = 0; k < 2 * K; k++) c[k] = fe_zero();
        } else if (ok) {
            Affine<F> a;
            for (int k = 0; k < 2 * K; k++) c[k] = to_mont(c[k]);
            as_elem(a.x, c); as_elem(a.y, c + K);
            ok = !C::aff_is_inf(a) && aff_on_curve<C, F>(a);   // (0, 0) without the infinity flag is off the curve
        }
    }
    if (!ok) {
        atomicMin(bad, (unsigned long long)(base + i));
        for (int k = 0; k < 2 * K; k++) c[k] = fe_zero();
    }
    for (int k = 0; k < 2 * K; k++) fe_store(pts + ((size_t)i * 2 * K + k) * 32, c[k]);
}

// G2 membership of every decoded point, one point per thread, in its own kernel so that the decoder does not carry
// g2_in_subgroup's registers and stack (as decompress_g2_kernel); points that did not decode are zeros and are skipped
__global__ void __launch_bounds__(128) points_g2_subgroup_kernel(const uint8_t* __restrict__ pts, uint32_t n, uint64_t base,
                                                                 unsigned long long* __restrict__ bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G2::Aff q = aff_load<Fq2>(pts, i);
    if (G2::aff_is_inf(q) || g2_in_subgroup(q)) return;
    // the index again from the special registers, so that no value has to live across the call
    atomicMin(bad, (unsigned long long)(base + blockIdx.x * blockDim.x + threadIdx.x));
}

// ---------------------------------------------------------------------------------------------- rerandomization
// b2g_rerandomize_many: ark-groth16 0.5.0's Groth16::rerandomize_proof for a proof (A, B, C) and nonzero factors r1, r2:
//     A' = r1^-1 A,   B' = r1 B + (r1 r2) delta_2,   C' = C + r2 A
// A scalar below r has at most RERAND_BITS bits.
constexpr int RERAND_BITS = 254;

// k1 b + k2 d for scalars below r (canonical): one doubling chain over both scalars (Shamir's trick), each step adding b, d
// or b + d, all three affine so that every addition is a mixed one; every exceptional case is left to madd
__device__ __noinline__ G2::Pt g2_joint_mul(const G2::Aff& b, const G2::Aff& d, const uint32_t* k1, const uint32_t* k2) {
    G2::Pt t = G2::from_affine(b);
    G2::madd(t, d);
    const G2::Aff bd = G2::to_affine(t);
    G2::Pt acc = G2::infinity();
    #pragma unroll 1
    for (int i = RERAND_BITS - 1; i >= 0; i--) {
        acc = G2::dbl(acc);
        const uint32_t u = (k1[i >> 5] >> (i & 31)) & 1u, v = (k2[i >> 5] >> (i & 31)) & 1u;
        if (u & v) G2::madd(acc, bd);
        else if (u) G2::madd(acc, b);
        else if (v) G2::madd(acc, d);
    }
    return acc;
}

// one proof per thread: row j of proofs (b2g_prove layout) with the factors r1[j], r2[j] (canonical, nonzero, below r: the
// host checks them) -> the canonical rerandomized row j of out and ok[j] = 1, or the 0xFF row and ok[j] = 0 when row j does
// not parse (a coordinate >= p or a point off its curve: proof_parse, the rule of b2g_verify_many).  delta = delta_2 (affine
// Montgomery, zeros = infinity).  No G2 subgroup check, as in arkworks.
__global__ void __launch_bounds__(64) rerandomize_kernel(const uint8_t* __restrict__ proofs, const uint8_t* __restrict__ r1s,
                                                         const uint8_t* __restrict__ r2s, const uint8_t* __restrict__ delta,
                                                         uint32_t count, uint8_t* __restrict__ out, uint8_t* __restrict__ ok) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    G1::Aff a, cc; G2::Aff b;
    const bool good = proof_parse(proofs + (size_t)j * 256, a, b, cc);
    ok[j] = good;
    if (!good) { coords_store(out + (size_t)j * 256, nullptr, 8, false); return; }
    const fe r1 = fe_load(r1s + (size_t)j * 32), r2 = fe_load(r2s + (size_t)j * 32);
    const fe r1m = Fr::from_canonical(r1);
    const fe r1_inv = Fr::to_canonical(Fr::inv(r1m));
    const fe r12 = Fr::mul(r1m, r2);                     // r1 R r2 / R: canonical r1 r2 mod r
    const G1::Aff a2 = G1::to_affine(G1::mul_affine(a, r1_inv.l, 8));
    G1::Pt c2 = G1::mul_affine(a, r2.l, 8);
    G1::madd(c2, cc);
    const G2::Aff b2 = G2::to_affine(g2_joint_mul(b, aff_load<Fq2>(delta, 0), r1.l, r12.l));
    const G1::Aff c2a = G1::to_affine(c2);
    fe c[8] = {a2.x, a2.y, b2.x.c0, b2.x.c1, b2.y.c0, b2.y.c1, c2a.x, c2a.y};
    for (int k = 0; k < 8; k++) c[k] = Fq::to_canonical(c[k]);
    coords_store(out + (size_t)j * 256, c, 8, true);
}

// ---------------------------------------------------------------------------------------------- key preparation
// b2g_vk_load_many (b2g_vk_load is its call of one key) prepares every key of a call in four launches, whatever the number
// of keys and of public inputs; each kernel finds its key in the call's VkRec table.

// one thread per point of every key: key k's points are its G1 points alpha, IC[0..n_public], then its G2 points beta,
// gamma, delta.  bad[2k] (G1) and bad[2k + 1] (G2) receive 1 + the greatest index of an off-curve point among them, the
// index msm_validate_points reports.
__global__ void __launch_bounds__(256) vk_validate_kernel(const VkRec* __restrict__ keys, uint32_t n_keys, uint64_t n_pts,
                                                          uint32_t* __restrict__ bad) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_pts) return;
    const uint32_t k = seg_find<&VkRec::pt>(keys, n_keys, t);
    const VkRec& key = keys[k];
    const uint32_t j = (uint32_t)(t - key.pt), n_g1 = key.n_public + 2;
    if (j < n_g1) {
        if (!aff_on_curve<G1, Fq>(aff_load<Fq>(key.g1, j))) atomicMax(bad + 2 * k, j + 1);
    } else if (!aff_on_curve<G2, Fq2>(aff_load<Fq2>(key.g2, j - n_g1))) {
        atomicMax(bad + 2 * k + 1, j - n_g1 + 1);
    }
}

// e(alpha, beta) of every key, one key per thread
__global__ void __launch_bounds__(64) vk_pairing_kernel(const VkRec* __restrict__ keys, uint32_t n_keys) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_keys) return;
    fe12 e;
    pairing(e, aff_load<Fq>(keys[k].g1, 0), aff_load<Fq2>(keys[k].g2, 0));
    Fq12::store(keys[k].eab, e);
}

// the lines of -gamma (thread 2k) and -delta (thread 2k + 1) of key k for every loop step, in the order miller_loop reads
// them; nothing for a point at infinity, whose pair drops out
__global__ void __launch_bounds__(64) vk_lines_kernel(const VkRec* __restrict__ keys, uint32_t n_keys) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * (uint64_t)n_keys) return;
    const VkRec& key = keys[t >> 1];
    const uint32_t s = (uint32_t)(t & 1);
    const G2::Aff q = aff_load<Fq2>(key.g2, 1 + s);
    if (G2::aff_is_inf(q)) return;
    uint8_t* out = key.lines + (size_t)s * ATE_LINES * LINE_BYTES;
    g2_line_walk(q.x, Fq2::neg(q.y), [&](const fe2* c) {
        elem_store(out, c[0]); elem_store(out + 64, c[1]); elem_store(out + 128, c[2]);
        out += LINE_BYTES;
    });
}

// every window table of every key, one entry per thread: the tables of all keys are numbered back to back, and table t
// (key k's IC[j + 1], j = t - keys[k].tab) gets its entry e % TABLE_POINTS.  The points are indexed on grid.x, so the
// number of tables is not bound by a grid dimension.
__global__ void __launch_bounds__(64) vk_tables_kernel(const VkRec* __restrict__ keys, uint32_t n_keys, uint64_t n_entries) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    const uint64_t t = e / TABLE_POINTS;
    // a key without inputs shares its tab with the next key, so the last key with tab <= t is the one that holds t
    const VkRec& key = keys[seg_find<&VkRec::tab>(keys, n_keys, t)];
    const uint64_t j = t - key.tab;
    fixed_table_entry<G1, Fq>(key.tabs + j * TABLE_BYTES, key.g1 + (2 + j) * 64, (uint32_t)(e % TABLE_POINTS));
}

// b2g_test_op ops 30-42 on Fq12 values (384 B), G1 / G2 affine points (64 / 128 B), lines (3 Fq2, 192 B) and projective
// twist points (X, Y, Z: 192 B), Montgomery
__global__ void pairing_test_kernel(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe12 r;
    if (op == 37) {
        pairing(r, aff_load<Fq>(a, i), aff_load<Fq2>(b, i));
    } else if (op == 40) {
        const G1::Aff p = aff_load<Fq>(a, i);
        const G2::Aff q = aff_load<Fq2>(b, i);
        miller_loop(r, !G1::aff_is_inf(p) && !G2::aff_is_inf(q), p, q, 0, nullptr, nullptr);
    } else if (op == 41 || op == 42) {                     // one line step: out = T' (192 B) || (c0, c1, c2) (192 B)
        G2Proj t;
        const uint8_t* tp = a + (size_t)i * LINE_BYTES;
        elem_load(t.x, tp); elem_load(t.y, tp + 64); elem_load(t.z, tp + 128);
        fe2 c[3];
        if (op == 41) line_dbl(t, c);
        else { const G2::Aff q = aff_load<Fq2>(b, i); line_add(t, q.x, q.y, c); }
        uint8_t* o = out + (size_t)i * F12_BYTES;
        elem_store(o, t.x); elem_store(o + 64, t.y); elem_store(o + 128, t.z);
        for (int k = 0; k < 3; k++) elem_store(o + 192 + 64 * k, c[k]);
        return;
    } else {
        const fe12 x = Fq12::load(a + (size_t)i * F12_BYTES);
        switch (op) {
            case 30: Fq12::mul(r, x, Fq12::load(b + (size_t)i * F12_BYTES)); break;
            case 31: Fq12::sqr(r, x); break;
            case 32: Fq12::cyclotomic_sqr(r, x); break;
            case 33: case 34: case 35: Fq12::frobenius(r, x, op - 32); break;
            case 36: Fq12::final_exponentiation(r, x); break;
            case 38: Fq12::inv(r, x); break;
            default: {                                     // 39: x * (c0 + c3 w + c4 w^3)
                fe2 c[3];
                for (int k = 0; k < 3; k++) elem_load(c[k], b + (size_t)i * LINE_BYTES + 64 * k);
                r = x;
                Fq12::mul_by_034(r, c[0], c[1], c[2]);
            }
        }
    }
    Fq12::store(out + (size_t)i * F12_BYTES, r);
}

// ops 49-53 (see include/b2groth.h) run the kernels the verifier runs, not test copies of them: ptxas compiles each kernel
// with its own copy of the __noinline__ calls it reaches (miller_loop_t, ell_fixed, the tower), so only a launch of the
// shipped kernel tests the shipped machine code.  Per row of ops 49 and 53, a staging region holds the key's G2 points for
// vk_lines_kernel (an unused slot, gamma, delta), then the row's proof record (op 49) or batch tail (op 53), then the lines
// of -gamma and -delta; a point given as zeros is infinity and drops its pair, as in b2g_vk_load.  Ops 49, 50 and 52 make
// each row (or pair of rows) a key of one b2g_vk_load_many kernel launch.
constexpr size_t STAGE_G2 = 0, STAGE_REC = 384, STAGE_LINES = STAGE_REC + TAIL_BYTES, STAGE_BYTES = STAGE_LINES + 2 * ATE_LINES * LINE_BYTES;

static void verify_stage_test_op(cudaStream_t st, int op, const void* a, const void* b, size_t n, void* out) {
    if (op == 51 && !b) throw_error(B2G_E_SHAPE, "this op needs operand b");
    const size_t sa = op == 49 ? 576 : (op == 50 ? 128 : (op == 51 ? 32 : (op == 52 ? 64 : 512)));
    const size_t so = (op == 49 || op == 53) ? F12_BYTES : (op == 50 ? ATE_LINES * LINE_BYTES : (op == 51 ? 128 : TABLE_BYTES));
    if (n == 0) return;
    struct Bufs { uint8_t *a = nullptr, *s = nullptr, *o = nullptr; ~Bufs() { for (void* p : {(void*)a, (void*)s, (void*)o}) if (p) cudaFree(p); } } d;
    const uint8_t* in = (const uint8_t*)a;
    if (op == 49 || op == 53) {
        // op 49 row: A (64 B), B (128 B), the prepared inputs (64 B), C (64 B), gamma, delta (128 B each) -> a verify_many
        // record; op 53 row: the prepared inputs and sum r C (XYZZ, 128 B each), gamma, delta -> a verify_batch tail
        std::vector<uint8_t> stage(n * STAGE_BYTES, 0);
        std::vector<uint8_t> on(2 * n);
        for (size_t i = 0; i < n; i++) {
            const uint8_t* row = in + i * sa;
            uint8_t* g = stage.data() + i * STAGE_BYTES;
            const uint8_t* q = row + (op == 49 ? 320 : 256);
            memcpy(g + STAGE_G2 + 128, q, 256);
            on[2 * i] = !all_zero(q, 128);
            on[2 * i + 1] = !all_zero(q + 128, 128);
            uint8_t* r = g + STAGE_REC;
            if (op == 49) {
                memcpy(r, row, 64);                             // A
                memcpy(r + 64, row + 64, 128);                  // B
                memcpy(r + 192, row + 256, 64);                 // C
                memcpy(r + 256, row + 192, 64);                 // the prepared inputs
                *reinterpret_cast<uint32_t*>(r + REC_OK) = 1;
            } else {
                memcpy(r + TAIL_PREP, row, 128);
                memcpy(r + TAIL_RC, row + 128, 128);
            }
        }
        d.s = dev_upload<uint8_t>(stage.data(), stage.size(), st);
        CUDA_CHECK(cudaMalloc(&d.o, n * so));
        // per row, a key record with the row's lines and a one-segment table, as verify_many_enqueue and batch_enqueue build
        // them, then the rows as the keys of one vk_lines_kernel launch, as b2g_vk_load_many builds them
        std::vector<uint8_t> meta(n * sizeof(KeyRec) + sizeof(Seg) + n * sizeof(VkRec));
        KeyRec* keys = reinterpret_cast<KeyRec*>(meta.data());
        VkRec* vks = reinterpret_cast<VkRec*>(meta.data() + n * sizeof(KeyRec) + sizeof(Seg));
        for (size_t i = 0; i < n; i++) {
            uint8_t* g = d.s + i * STAGE_BYTES;
            keys[i] = {g + STAGE_LINES, nullptr, nullptr, nullptr, 0, on[2 * i], on[2 * i + 1], 0};
            vks[i] = {0, 0, nullptr, g + STAGE_G2, nullptr, g + STAGE_LINES, nullptr, 0, 0};
        }
        const Seg seg = {0, 0, 0, 1, 0, 1, 0};
        memcpy(meta.data() + n * sizeof(KeyRec), &seg, sizeof(Seg));
        d.a = dev_upload<uint8_t>(meta.data(), meta.size(), st);
        CUDA_CHECK(cudaStreamSynchronize(st));             // meta is pageable and leaves scope here
        const Seg* d_seg = (const Seg*)(d.a + n * sizeof(KeyRec));
        vk_lines_kernel<<<(unsigned)((2 * n + 63) / 64), 64, 0, st>>>((const VkRec*)(d.a + n * sizeof(KeyRec) + sizeof(Seg)), (uint32_t)n);
        for (size_t i = 0; i < n; i++) {
            uint8_t* g = d.s + i * STAGE_BYTES;
            if (op == 49) {
                verify_miller_kernel<<<1, 64, 0, st>>>(g + STAGE_REC, (const KeyRec*)d.a + i, d_seg, 1, 1, d.o + i * F12_BYTES);
            } else {
                batch_pairs_kernel<<<1, 1, 0, st>>>(g + STAGE_REC, 1, d_seg, (const KeyRec*)d.a + i);
                CUDA_CHECK(cudaMemcpyAsync(d.o + i * F12_BYTES, g + STAGE_REC + TAIL_G, F12_BYTES, cudaMemcpyDeviceToDevice, st));
            }
        }
        g_launch_count += 1 + n;
    } else if (op == 50) {
        // the lines of -a: rows 2k and 2k + 1 are the gamma and delta of key k of one vk_lines_kernel launch
        const size_t pairs = (n + 1) / 2;
        std::vector<uint8_t> g2(pairs * 384, 0);
        for (size_t i = 0; i < n; i++) memcpy(g2.data() + (i / 2) * 384 + 128 * (1 + i % 2), in + i * 128, 128);
        d.a = dev_upload<uint8_t>(g2.data(), g2.size(), st);
        CUDA_CHECK(cudaMalloc(&d.o, 2 * pairs * so));
        std::vector<VkRec> vks(pairs);
        for (size_t k = 0; k < pairs; k++) vks[k] = {0, 0, nullptr, d.a + k * 384, nullptr, d.o + 2 * k * so, nullptr, 0, 0};
        d.s = dev_upload<uint8_t>(vks.data(), pairs * sizeof(VkRec), st);
        CUDA_CHECK(cudaStreamSynchronize(st));             // vks is pageable and leaves scope here
        vk_lines_kernel<<<(unsigned)((2 * pairs + 63) / 64), 64, 0, st>>>((const VkRec*)d.s, (uint32_t)pairs);
        g_launch_count += 1;
    } else if (op == 51) {
        d.a = dev_upload<uint8_t>(a, n * sa, st);
        CUDA_CHECK(cudaMalloc(&d.o, n * so));
        // the point, a one-input key record and a one-segment table over the n rows, then the point's table
        CUDA_CHECK(cudaMalloc(&d.s, 256 + TABLE_BYTES));
        static_assert(128 + sizeof(KeyRec) + sizeof(Seg) <= 256, "the op 51 tables fit between the point and its table");
        uint8_t meta[256] = {};
        memcpy(meta, b, 64);
        const KeyRec key = {nullptr, nullptr, d.s + 256, nullptr, 1, 0, 0, 0};
        const Seg seg = {0, 0, 0, (uint32_t)n, 0, 0, 0};
        memcpy(meta + 128, &key, sizeof(KeyRec));
        memcpy(meta + 128 + sizeof(KeyRec), &seg, sizeof(Seg));
        CUDA_CHECK(cudaMemcpyAsync(d.s, meta, 256, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));             // meta is pageable and leaves scope here
        fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(d.s + 256, d.s);
        verify_inputs_kernel<<<(unsigned)((n + 3) / 4), 128, 0, st>>>((const KeyRec*)(d.s + 128), (const Seg*)(d.s + 128 + sizeof(KeyRec)), 1,
                                                                      (const uint32_t*)d.a, n, d.o);
        g_launch_count += 2;
    } else {
        // row i is IC[1] of key i of one vk_tables_kernel launch: its G1 slots are (unused alpha, unused IC[0], the row)
        std::vector<uint8_t> g1(n * 192, 0);
        for (size_t i = 0; i < n; i++) memcpy(g1.data() + i * 192 + 128, in + i * 64, 64);
        d.a = dev_upload<uint8_t>(g1.data(), g1.size(), st);
        CUDA_CHECK(cudaMalloc(&d.o, n * so));
        std::vector<VkRec> vks(n);
        for (size_t i = 0; i < n; i++) vks[i] = {0, i, d.a + i * 192, nullptr, nullptr, nullptr, d.o + i * TABLE_BYTES, 1, 0};
        d.s = dev_upload<uint8_t>(vks.data(), n * sizeof(VkRec), st);
        CUDA_CHECK(cudaStreamSynchronize(st));             // g1 and vks are pageable and leave scope here
        vk_tables_kernel<<<(unsigned)((n * TABLE_POINTS + 63) / 64), 64, 0, st>>>((const VkRec*)d.s, (uint32_t)n, (uint64_t)n * TABLE_POINTS);
        g_launch_count += 1;
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d.o, n * so, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

void pairing_test_op(cudaStream_t st, int op, const void* a, const void* b, size_t n, void* out) {
    if (op > 53 || !a || !out) throw_error(B2G_E_SHAPE, "bad arguments");
    if (op >= 49) { verify_stage_test_op(st, op, a, b, n, out); return; }
    const bool batch_op = op >= 43 && op <= 45, decompress_op = op >= 46;
    size_t sa = (op == 37 || op == 40) ? 64 : ((op == 41 || op == 42) ? LINE_BYTES : F12_BYTES);
    size_t sb = op == 30 ? F12_BYTES : ((op == 37 || op == 40 || op == 42) ? 128 : (op == 39 ? LINE_BYTES : 0));
    size_t so = F12_BYTES;
    if (op == 43) { sa = 128; sb = 0; so = 8; }
    if (op == 44) { sa = 64; sb = 16; so = 64; }
    if (op == 45) { sa = F12_BYTES; sb = 32; so = F12_BYTES; }
    if (op == 46) { sa = 32; sb = 0; so = 64; }
    if (op == 47) { sa = 64; sb = 0; so = 96; }
    if (op == 48) { sa = 64; sb = 0; so = 160; }
    if (sb && !b) throw_error(B2G_E_SHAPE, "this op needs operand b");
    if (n == 0) return;
    struct Bufs { uint8_t *a = nullptr, *b = nullptr, *o = nullptr; ~Bufs() { for (void* p : {(void*)a, (void*)b, (void*)o}) if (p) cudaFree(p); } } d;
    d.a = dev_upload<uint8_t>(a, n * sa, st);
    if (sb) d.b = dev_upload<uint8_t>(b, n * sb, st);
    CUDA_CHECK(cudaMalloc(&d.o, n * so));
    if (batch_op) batch_test_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(op, d.a, d.b, (uint32_t)n, d.o);
    else if (decompress_op) decompress_test_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(op, d.a, (uint32_t)n, d.o);
    else pairing_test_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(op, d.a, d.b, (uint32_t)n, d.o);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d.o, n * so, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ------------------------------------------------------------------------------------------------ host side
// grows one of the context's verification buffers to `bytes`; never shrinks it.  The buffer is marked empty before it is
// reallocated, so a failed allocation leaves the context consistent.
static void vbuf_grow(uint8_t*& p, size_t& cap, size_t bytes) {
    if (bytes <= cap) return;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    CUDA_CHECK(cudaMalloc(&p, bytes));
    cap = bytes;
}

// grows the context's verification buffers to `count` proofs, `inputs` public-input scalars, `parts` (proof, input) G1
// records, `batch` bytes of b2g_verify_batch scratch, `comp` bytes of compressed-proof staging and `meta` bytes of
// b2g_verify_many tables; never shrinks them, and a failed allocation leaves them consistent
static void vbufs_ensure(VerifyBufs*& v, size_t count, size_t inputs, size_t parts, size_t batch = 0, size_t comp = 0, size_t meta = 0) {
    if (!v) v = new VerifyBufs();
    if (count > v->cap_count) {
        for (uint8_t** p : {&v->d_proofs, &v->d_rec, &v->d_f, &v->d_verdict}) { if (*p) cudaFree(*p); *p = nullptr; }
        v->cap_count = 0;
        CUDA_CHECK(cudaMalloc(&v->d_proofs, count * 256));
        CUDA_CHECK(cudaMalloc(&v->d_rec, count * REC_BYTES_V));
        CUDA_CHECK(cudaMalloc(&v->d_f, count * F12_BYTES));
        CUDA_CHECK(cudaMalloc(&v->d_verdict, count));
        v->cap_count = count;
    }
    vbuf_grow(v->d_pub, v->cap_pub, inputs * 32);
    vbuf_grow(v->d_part, v->cap_part, parts * 128);
    vbuf_grow(v->d_batch, v->cap_batch, batch);
    vbuf_grow(v->d_comp, v->cap_comp, comp);
    vbuf_grow(v->d_meta, v->cap_meta, meta);
}

// the staging bytes of count compressed proofs: the rows, then one ok byte per proof
static size_t comp_bytes(uint32_t count) { return (size_t)count * (COMP_BYTES + 1); }

// uploads count compressed proofs to the staging buffer and decodes them into v.d_proofs on st; with g2_check, a decoded B
// outside G2 also turns its row into the 0xFF row.  Returns the device ok bytes.
static uint8_t* decompress_enqueue(VerifyBufs& v, const void* compressed, uint32_t count, bool g2_check, cudaStream_t st) {
    uint8_t* ok = v.d_comp + (size_t)count * COMP_BYTES;
    CUDA_CHECK(cudaMemcpyAsync(v.d_comp, compressed, (size_t)count * COMP_BYTES, cudaMemcpyHostToDevice, st));
    decompress_kernel<<<(count + 127) / 128, 128, 0, st>>>(v.d_comp, count, v.d_proofs, ok);
    if (g2_check) decompress_g2_kernel<<<(count + 127) / 128, 128, 0, st>>>(count, v.d_proofs, ok);
    g_launch_count += g2_check ? 2 : 1;
    return ok;
}

// the two side streams and six events of the batch check (batch_enqueue), created at the first such call on the context.  The
// side streams have the greatest priority, so that their tail kernels are scheduled ahead of queued per-proof CTAs.
static void batch_streams(VerifyBufs& v) {
    if (v.ev[5]) return;
    int least = 0, greatest = 0;
    CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    for (cudaStream_t& s : v.side) if (!s) CUDA_CHECK(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, greatest));
    for (cudaEvent_t& e : v.ev) if (!e) CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
}

// the CTAs of a segmented reduction to one value per segment, `per` records per CTA, level by level: the first level reads
// each segment's records (segs[k].first .. + count), each later level the values the previous level wrote for the segments
// that still have more than one, and a segment's last value goes to its tail.  Appends the spans of every level to `spans`
// and returns the number of CTAs per level; *scratch = the most values one level writes below the tails.
static std::vector<uint32_t> reduce_plan(const std::vector<Seg>& segs, uint32_t per, std::vector<Span>& spans, size_t* scratch) {
    std::vector<uint32_t> first(segs.size()), len(segs.size()), levels;
    for (size_t k = 0; k < segs.size(); k++) { first[k] = segs[k].first; len[k] = segs[k].count; }
    for (uint32_t out = 1; out;) {
        const size_t before = spans.size();
        out = 0;
        for (uint32_t k = 0; k < (uint32_t)segs.size(); k++) {
            if (!len[k]) continue;                         // done at an earlier level
            const uint32_t blocks = (len[k] + per - 1) / per;
            for (uint32_t b = 0; b < blocks; b++)
                spans.push_back({first[k] + b * per, std::min(per, len[k] - b * per), blocks == 1 ? TO_TAIL | k : out + b});
            if (blocks == 1) { len[k] = 0; continue; }
            first[k] = out; len[k] = blocks; out += blocks;
        }
        levels.push_back((uint32_t)(spans.size() - before));
        *scratch = std::max(*scratch, (size_t)out);
    }
    return levels;
}

// launches the levels of a reduce_plan: the first reads `src` (`stride` bytes apart) under the mask, the later ones the
// scratch areas x and y in turn (rec_bytes apart); level(blocks, src, stride, spans, mask, dst) launches one level
template <class Level>
static void reduce_run(const std::vector<uint32_t>& levels, const Span* spans, const uint8_t* src, size_t stride, size_t rec_bytes,
                       const uint8_t* mask, uint8_t* x, uint8_t* y, Level&& level) {
    for (uint32_t blocks : levels) {
        level(blocks, src, stride, spans, mask, x);
        g_launch_count += 1;
        spans += blocks; src = x; stride = rec_bytes; mask = nullptr;
        std::swap(x, y);
    }
}

// one segment of the batch check: `count` consecutive proofs under key record `key`
struct SegIn { uint32_t key, count; };

// b2g_vk_load_many: the checks, one allocation carved into every key's arrays (each 256-byte aligned), one upload of every
// key's points and of the VkRec table, the on-curve checks and one synchronise, then e(alpha, beta), the lines and the window
// tables of every key in three launches and a second synchronise.  The handles are made only once everything succeeded.
// b2g_vk_load is the call of one key (`one`): its messages keep their form without a key index.
static void vk_load_many(b2g_ctx* ctx, uint32_t n_keys, const b2g_vk_desc* descs, b2g_vk** out, bool one) {
    static const char* fn = "b2g_vk_load_many";
    auto at = [&](uint32_t k) { return one ? std::string() : std::string(fn) + ": key " + std::to_string(k) + ": "; };
    if (!ctx || !descs || !out) throw_error(B2G_E_SHAPE, one ? "null pointer" : std::string(fn) + ": null pointer");
    if (n_keys == 0) throw_error(B2G_E_SHAPE, std::string(fn) + ": n_keys must be at least 1");
    for (uint32_t k = 0; k < n_keys; k++) {
        const b2g_vk_desc& d = descs[k];
        if (!d.alpha_g1 || !d.beta_g2 || !d.gamma_g2 || !d.delta_g2 || !d.gamma_abc_g1) throw_error(B2G_E_SHAPE, at(k) + "null verifying-key field");
    }
    const CtxView cv = ctx_view(ctx);
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    // the layout: the uploaded part first (per key its G1 points alpha, IC[0..n_public] and its G2 points beta, gamma, delta;
    // then the VkRec table), then the on-curve status words, then per key e(alpha, beta), the lines and the window tables
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    static_assert(TABLE_BYTES % 256 == 0, "window tables stay 256-byte aligned");
    std::vector<size_t> o_g1(n_keys), o_g2(n_keys), o_eab(n_keys);
    size_t o = 0;
    uint64_t n_pts = 0, n_tabs = 0;
    for (uint32_t k = 0; k < n_keys; k++) {
        o_g1[k] = o; o += up(((size_t)descs[k].n_public + 2) * 64);
        o_g2[k] = o; o += up(3 * 128);
        n_pts += (uint64_t)descs[k].n_public + 5; n_tabs += descs[k].n_public;
    }
    const size_t o_recs = o, n_up = o + (size_t)n_keys * sizeof(VkRec);
    const size_t o_bad = up(n_up);
    o = o_bad + up((size_t)n_keys * 8);
    for (uint32_t k = 0; k < n_keys; k++) { o_eab[k] = o; o += up(F12_BYTES) + up(2 * ATE_LINES * LINE_BYTES) + descs[k].n_public * TABLE_BYTES; }
    auto arena = std::make_shared<VkArena>();
    if (cudaMalloc(&arena->base, o) != cudaSuccess) {
        cudaGetLastError();
        arena->base = nullptr;
        throw_error(B2G_E_DEVICE, std::string(fn) + ": the device state of " + std::to_string(n_keys) + (n_keys == 1 ? " key (" : " keys (") +
                                  std::to_string((o + (1 << 20) - 1) >> 20) + " MiB) does not fit in device memory");
    }
    uint8_t* base = arena->base;
    std::vector<uint8_t> h(n_up, 0);
    VkRec* recs = reinterpret_cast<VkRec*>(h.data() + o_recs);
    uint64_t pt = 0, tab = 0;
    for (uint32_t k = 0; k < n_keys; k++) {
        const b2g_vk_desc& d = descs[k];
        uint8_t *g1 = h.data() + o_g1[k], *g2 = h.data() + o_g2[k];
        memcpy(g1, d.alpha_g1, 64);
        memcpy(g1 + 64, d.gamma_abc_g1, ((size_t)d.n_public + 1) * 64);
        memcpy(g2, d.beta_g2, 128); memcpy(g2 + 128, d.gamma_g2, 128); memcpy(g2 + 256, d.delta_g2, 128);
        uint8_t* eab = base + o_eab[k];
        recs[k] = {pt, tab, base + o_g1[k], base + o_g2[k], eab, eab + up(F12_BYTES),
                   d.n_public ? eab + up(F12_BYTES) + up(2 * ATE_LINES * LINE_BYTES) : nullptr, d.n_public, 0};
        pt += (uint64_t)d.n_public + 5; tab += d.n_public;
    }
    const VkRec* d_recs = reinterpret_cast<const VkRec*>(base + o_recs);
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(base + o_bad);
    std::vector<uint32_t> bad(2 * (size_t)n_keys);
    try {
        // prepare_verifying_key checks every point (verifier.py): an off-curve point fails the call with B2G_E_INPUT, naming the
        // lowest key that holds one and, as msm_validate_points does, its G1 points before its G2 points
        CUDA_CHECK(cudaMemcpyAsync(base, h.data(), n_up, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemsetAsync(d_bad, 0, (size_t)n_keys * 8, st));
        vk_validate_kernel<<<(unsigned)((n_pts + 255) / 256), 256, 0, st>>>(d_recs, n_keys, n_pts, d_bad);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(bad.data(), d_bad, (size_t)n_keys * 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        for (uint32_t k = 0; k < n_keys; k++) {
            if (bad[2 * k]) throw_error(B2G_E_INPUT, at(k) + "G1 point " + std::to_string(bad[2 * k] - 1) + " of alpha_g1 / gamma_abc_g1 is not on the curve");
            if (bad[2 * k + 1]) throw_error(B2G_E_INPUT, at(k) + "G2 point " + std::to_string(bad[2 * k + 1] - 1) + " of beta_g2 / gamma_g2 / delta_g2 is not on the curve");
        }
        // the table kernel is launched without tables too (one CTA that does nothing), so that the launches do not depend on
        // the public-input counts
        const uint64_t entries = n_tabs * TABLE_POINTS;
        vk_pairing_kernel<<<(n_keys + 63) / 64, 64, 0, st>>>(d_recs, n_keys);
        vk_lines_kernel<<<(unsigned)((2 * (uint64_t)n_keys + 63) / 64), 64, 0, st>>>(d_recs, n_keys);
        vk_tables_kernel<<<(unsigned)std::max<uint64_t>(1, (entries + 63) / 64), 64, 0, st>>>(d_recs, n_keys, entries);
        g_launch_count += 3;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(st));
    } catch (...) {
        cudaDeviceSynchronize();                           // nothing may still use the allocation when it is freed
        throw;
    }
    std::vector<std::unique_ptr<b2g_vk>> vks(n_keys);
    for (uint32_t k = 0; k < n_keys; k++) {
        const VkRec& r = recs[k];
        vks[k].reset(new b2g_vk());
        b2g_vk* vk = vks[k].get();
        vk->device = cv.device; vk->n_public = descs[k].n_public; vk->arena = arena;
        vk->d_g1 = r.g1; vk->d_g2 = r.g2; vk->d_eab = r.eab; vk->d_lines = r.lines; vk->d_tabs = r.tabs;
        vk->gamma_inf = all_zero(descs[k].gamma_g2, 128);
        vk->delta_inf = all_zero(descs[k].delta_g2, 128);
    }
    for (uint32_t k = 0; k < n_keys; k++) out[k] = vks[k].release();
}

// the slice loop of b2g_points_serialize / b2g_points_deserialize: one device allocation of min(n, KEY_SLICE) input rows,
// as many output rows and the bad-index word, reused by every slice.  Per slice: the upload, run(d_in, d_out, count, base,
// d_bad, st), the download and one synchronise; a slice with a bad point ends the loop, as no later point can be lower.
// Returns the lowest bad index, or n.
template <class Run>
static uint64_t points_slices(const char* fn, b2g_ctx* ctx, size_t n, size_t in_row, size_t out_row, const void* in, void* out, Run&& run) {
    const CtxView cv = ctx_idle(ctx);
    if (n == 0) return 0;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    const size_t slice = std::min(n, KEY_SLICE), bytes = slice * (in_row + out_row) + 8;
    DevArena mem(st);
    uint8_t* d_in = nullptr;
    try {
        d_in = mem.alloc(bytes);
    } catch (const B2gError&) {
        cudaGetLastError();
        throw_error(B2G_E_DEVICE, std::string(fn) + ": the device buffer of " + std::to_string(slice) + " points (" +
                                  std::to_string((bytes + (1 << 20) - 1) >> 20) + " MiB) does not fit in device memory");
    }
    uint8_t* d_out = d_in + slice * in_row;
    unsigned long long* d_bad = reinterpret_cast<unsigned long long*>(d_out + slice * out_row);
    uint64_t bad = n;
    CUDA_CHECK(cudaMemcpyAsync(d_bad, &bad, 8, cudaMemcpyHostToDevice, st));
    for (size_t base = 0; base < n && bad == n; base += slice) {
        const size_t m = std::min(slice, n - base);
        CUDA_CHECK(cudaMemcpyAsync(d_in, (const uint8_t*)in + base * in_row, m * in_row, cudaMemcpyHostToDevice, st));
        run(d_in, d_out, (uint32_t)m, (uint64_t)base, d_bad, st);
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync((uint8_t*)out + base * out_row, d_out, m * out_row, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    }
    return bad;
}

// b2g_setup's generators: bad[0] for g1 (thread 0), bad[1] for g2 (thread 1), with the codes of setup_generators_check
__global__ void setup_generators_kernel(const void* __restrict__ g1, const void* __restrict__ g2, uint32_t* __restrict__ bad) {
    if (threadIdx.x == 0 && g1) {
        const G1::Aff p = aff_load<Fq>(g1, 0);
        bad[0] = G1::aff_is_inf(p) || !aff_on_curve<G1, Fq>(p) ? 1u : 0u;
    } else if (threadIdx.x == 1 && g2) {
        const G2::Aff q = aff_load<Fq2>(g2, 0);
        bad[1] = G2::aff_is_inf(q) || !aff_on_curve<G2, Fq2>(q) ? 2u : (g2_in_subgroup(q) ? 0u : 3u);
    }
}

// bad = the lowest base + i whose point has a coordinate >= p or lies off its curve (infinity = zeros passes)
template <class C, class F>
__global__ void __launch_bounds__(128) points_curve_kernel(const uint8_t* __restrict__ pts, uint32_t n, uint64_t base,
                                                           unsigned long long* __restrict__ bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr int WORDS = 2 * Bytes<F>::ELEM / 32;
    bool ok = true;
    for (int k = 0; k < WORDS; k++) ok &= fe_below_p(fe_load(pts + ((size_t)i * WORDS + k) * 32));
    if (!ok || !aff_on_curve<C, F>(aff_load<F>(pts, i))) atomicMin(bad, (unsigned long long)(base + i));
}

uint64_t points_check(bool g2, const void* pts, size_t n, bool subgroup, cudaStream_t st, int* why) {
    *why = 0;
    if (n == 0) return 0;
    unsigned long long* d_bad = nullptr;
    CUDA_CHECK(cudaMalloc(&d_bad, 2 * sizeof(unsigned long long)));
    uint64_t bad[2] = {n, n};
    const unsigned blocks = (unsigned)((n + 127) / 128);
    cudaError_t e = cudaMemcpyAsync(d_bad, bad, sizeof(bad), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        if (g2) points_curve_kernel<G2, Fq2><<<blocks, 128, 0, st>>>((const uint8_t*)pts, (uint32_t)n, 0, d_bad);
        else points_curve_kernel<G1, Fq><<<blocks, 128, 0, st>>>((const uint8_t*)pts, (uint32_t)n, 0, d_bad);
        if (g2 && subgroup) points_g2_subgroup_kernel<<<blocks, 128, 0, st>>>((const uint8_t*)pts, (uint32_t)n, 0, d_bad + 1);
        g_launch_count += g2 && subgroup ? 2 : 1;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d_bad);
    CUDA_CHECK(e);
    // a point off its curve is also tested for G2 membership: the curve failure names it
    if (bad[0] < n && bad[0] <= bad[1]) { *why = 1; return bad[0]; }
    if (bad[1] < n) { *why = 2; return bad[1]; }
    return n;
}

// ---------------------------------------------------------------------------------------------- powers-of-tau point rules
// the first rule the affine point p (raw words at w) breaks, in b2g_powers_check's order: 1 a coordinate >= p, 2 off its curve,
// 3 at infinity, 4 outside G2 (only with `subgroup`), 5 not the generator (only with `gen`); 0 when it passes
template <class C, class F>
__device__ __forceinline__ uint32_t powers_rule(const uint8_t* w, bool gen, bool subgroup) {
    constexpr int WORDS = 2 * Bytes<F>::ELEM / 32;
    bool below = true;
    for (int k = 0; k < WORDS; k++) below &= fe_below_p(fe_load(w + 32 * k));
    if (!below) return 1;
    const typename C::Aff p = aff_load<F>(w, 0);
    if (!aff_on_curve<C, F>(p)) return 2;
    if (C::aff_is_inf(p)) return 3;
    if constexpr (std::is_same<F, Fq2>::value) { if (subgroup && !g2_in_subgroup(p)) return 4; }
    if (gen) {
        const typename C::Aff g = Gen<C>::get();
        if (!F::eq(p.x, g.x) || !F::eq(p.y, g.y)) return 5;
    }
    return 0;
}

// bad = the lowest base + i whose point breaks a rule other than G2 membership; `gen`: point 0 of the array must be the generator
template <class C, class F>
__global__ void __launch_bounds__(128) powers_rules_kernel(const uint8_t* __restrict__ pts, uint32_t n, uint64_t base, int gen,
                                                           unsigned long long* __restrict__ bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (powers_rule<C, F>(pts + (size_t)i * 2 * Bytes<F>::ELEM, gen && base + i == 0, false))
        atomicMin(bad, (unsigned long long)(base + i));
}

// *rule = the rule the one point at pt breaks (0: none)
template <class C, class F>
__global__ void powers_rule_kernel(const uint8_t* __restrict__ pt, int gen, uint32_t* __restrict__ rule) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *rule = powers_rule<C, F>(pt, gen != 0, true);
}

void powers_rules(bool g2, const void* pts, uint32_t n, uint64_t base, bool gen, unsigned long long* bad, cudaStream_t st) {
    if (n == 0) return;
    const unsigned blocks = (n + 127) / 128;
    if (g2) {
        powers_rules_kernel<G2, Fq2><<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, gen ? 1 : 0, bad);
        points_g2_subgroup_kernel<<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, bad);
    } else {
        powers_rules_kernel<G1, Fq><<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, gen ? 1 : 0, bad);
    }
    g_launch_count += g2 ? 2 : 1;
    CUDA_CHECK(cudaGetLastError());
}

uint32_t powers_point_rule(bool g2, const void* pt, bool gen, uint32_t* scratch, cudaStream_t st) {
    if (g2) powers_rule_kernel<G2, Fq2><<<1, 1, 0, st>>>((const uint8_t*)pt, gen ? 1 : 0, scratch);
    else powers_rule_kernel<G1, Fq><<<1, 1, 0, st>>>((const uint8_t*)pt, gen ? 1 : 0, scratch);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    uint32_t rule = 0;
    CUDA_CHECK(cudaMemcpyAsync(&rule, scratch, 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    return rule;
}

__device__ __forceinline__ G1::Pt g1_at(const uint8_t* g1, int k) { return G1::from_affine(aff_load<Fq>(g1, k)); }

// b2g_powers_check's pairing product, one block of 32 threads: *verdict = 1 iff the five-pair product of include/b2groth.h is 1.
// sums = S_T, S_A, S_B (G1 XYZZ), S_U (G2 XYZZ); g1 = T_0, T_1, T_(2n-2), A_0, A_(n-1), B_0, B_(n-1); g2 = U_0, U_1, U_(n-1),
// beta_2 (affine); ch = rho, sigma, pi, kappa, eps (canonical).  The products run on 11 threads, the Miller loops on 5.
__global__ void __launch_bounds__(32) powers_verdict_kernel(const uint8_t* __restrict__ sums, const uint8_t* __restrict__ g1,
                                                            const uint8_t* __restrict__ g2, const fe* __restrict__ ch, uint32_t log_n,
                                                            uint32_t* __restrict__ verdict) {
    __shared__ fe sc[3];                        // rho^(n-1), rho^(2n-2), kappa rho (canonical)
    __shared__ G1::Pt p1[11];
    __shared__ G2::Pt p2[2];
    __shared__ G1::Aff a1[5];
    __shared__ G2::Aff a2[2];
    __shared__ fe12 f[5];
    const uint32_t t = threadIdx.x;
    if (t == 0) {
        const fe rho = Fr::from_canonical(ch[0]);
        fe pw = Fr::one(), sq = rho;
        for (uint32_t e = (1u << log_n) - 1; e; e >>= 1) {
            if (e & 1) pw = Fr::mul(pw, sq);
            sq = Fr::sqr(sq);
        }
        sc[0] = Fr::to_canonical(pw);
        sc[1] = Fr::to_canonical(Fr::sqr(pw));
        sc[2] = Fr::to_canonical(Fr::mul(Fr::from_canonical(ch[3]), rho));
    }
    __syncthreads();
    const G1::Pt st = pt_load<Fq>(sums, 0), sa = pt_load<Fq>(sums, 1), sb = pt_load<Fq>(sums, 2);
    const G2::Pt su = pt_load<Fq2>(sums + 384, 0);
    // the products: p1 = X_T, X_A, X_B, kappa T_0, -kappa rho T_1, -eps T_0, eps B_0, sigma (S_A - A_0), pi (S_B - B_0); p2 = Q4, Q3
    if (t == 0) { G1::Pt r = st; G1::add(r, G1::neg(G1::mul_scalar(g1_at(g1, 2), sc[1].l))); p1[0] = r; }
    else if (t == 1) { G1::Pt r = sa; G1::add(r, G1::neg(G1::mul_scalar(g1_at(g1, 4), sc[0].l))); p1[1] = r; }
    else if (t == 2) { G1::Pt r = sb; G1::add(r, G1::neg(G1::mul_scalar(g1_at(g1, 6), sc[0].l))); p1[2] = r; }
    else if (t == 3) p1[3] = G1::mul_scalar(g1_at(g1, 0), ch[3].l);
    else if (t == 4) p1[4] = G1::neg(G1::mul_scalar(g1_at(g1, 1), sc[2].l));
    else if (t == 5) p1[5] = G1::neg(G1::mul_scalar(g1_at(g1, 0), ch[4].l));
    else if (t == 6) p1[6] = G1::mul_scalar(g1_at(g1, 5), ch[4].l);
    else if (t == 7) { G1::Pt r = sa; G1::add(r, G1::neg(g1_at(g1, 3))); p1[7] = G1::mul_scalar(r, ch[1].l); }
    else if (t == 8) { G1::Pt r = sb; G1::add(r, G1::neg(g1_at(g1, 5))); p1[8] = G1::mul_scalar(r, ch[2].l); }
    else if (t == 9) {
        G2::Pt r = su;
        G2::add(r, G2::neg(G2::mul_scalar(G2::from_affine(aff_load<Fq2>(g2, 2)), sc[0].l)));
        p2[0] = r;
    } else if (t == 10) { G2::Pt r = su; G2::add(r, G2::neg(G2::from_affine(aff_load<Fq2>(g2, 0)))); p2[1] = r; }
    __syncthreads();
    if (t == 0) p1[9] = G1::mul_scalar(p1[1], ch[1].l);                   // sigma X_A
    else if (t == 1) p1[10] = G1::mul_scalar(p1[2], ch[2].l);             // pi X_B
    __syncthreads();
    if (t == 0) {
        G1::Pt hi = st;                                                    // P_hi
        G1::add(hi, G1::neg(g1_at(g1, 0)));
        G1::add(hi, p1[7]); G1::add(hi, p1[8]); G1::add(hi, p1[6]);
        a1[0] = G1::to_affine(hi);
    } else if (t == 1) {
        G1::Pt lo = p1[0];                                                 // -P_lo
        G1::add(lo, p1[9]); G1::add(lo, p1[10]);
        a1[1] = G1::to_affine(G1::neg(G1::mul_scalar(lo, ch[0].l)));
    } else if (t >= 2 && t < 5) {
        a1[t] = G1::to_affine(p1[t + 1]);                                  // kappa T_0, -kappa rho T_1, -eps T_0
    } else if (t == 5) {
        a2[0] = G2::to_affine(p2[1]);                                      // S_U - U_0
    } else if (t == 6) {
        a2[1] = G2::to_affine(p2[0]);                                      // S_U - rho^(n-1) U_(n-1)
    }
    __syncthreads();
    if (t < 5) {
        G2::Aff q;
        if (t == 0) q = aff_load<Fq2>(g2, 0);
        else if (t == 1) q = aff_load<Fq2>(g2, 1);
        else if (t == 2) q = a2[0];
        else if (t == 3) q = a2[1];
        else q = aff_load<Fq2>(g2, 3);
        fe12 r;
        miller_loop(r, !G1::aff_is_inf(a1[t]) && !G2::aff_is_inf(q), a1[t], q, 0, nullptr, nullptr);
        f[t] = r;
    }
    __syncthreads();
    if (t == 0) {
        fe12 prod = f[0], e;
        for (int k = 1; k < 5; k++) Fq12::mul(prod, prod, f[k]);
        Fq12::final_exponentiation(e, prod);
        *verdict = Fq12::eq(e, Fq12::one()) ? 1u : 0u;
    }
}

void powers_verdict(const void* sums, const void* g1, const void* g2, const void* ch, uint32_t log_n, uint32_t* verdict, cudaStream_t st) {
    powers_verdict_kernel<<<1, 32, 0, st>>>((const uint8_t*)sums, (const uint8_t*)g1, (const uint8_t*)g2, (const fe*)ch, log_n, verdict);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- proving-key check
void setup_rules(bool g2, const void* pts, uint32_t n, uint64_t base, unsigned long long* bad, cudaStream_t st) {
    if (n == 0) return;
    const unsigned blocks = (n + 127) / 128;
    if (g2) {
        points_curve_kernel<G2, Fq2><<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, bad);
        points_g2_subgroup_kernel<<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, bad);
    } else {
        points_curve_kernel<G1, Fq><<<blocks, 128, 0, st>>>((const uint8_t*)pts, n, base, bad);
    }
    g_launch_count += g2 ? 2 : 1;
    CUDA_CHECK(cudaGetLastError());
}

// b2g_setup_check's equations, one block of 32 threads: *verdict = the lowest failing equation (1-6), or 0.  E1-E3 compare the
// XYZZ sums; the seven Miller loops of E4-E6 run on seven threads and the three final exponentiations on three.
__global__ void __launch_bounds__(32) setup_check_verdict_kernel(const uint8_t* __restrict__ sums, const uint8_t* __restrict__ g1,
                                                                 const uint8_t* __restrict__ g2, uint32_t* __restrict__ verdict) {
    __shared__ G1::Aff a1[7];
    __shared__ G2::Aff a2[7];
    __shared__ fe12 f[7];
    __shared__ uint32_t good[6];
    const uint32_t t = threadIdx.x;
    if (t == 0) good[0] = G1::pt_eq(pt_load<Fq>(sums + SC_KA, 0), pt_load<Fq>(sums + SC_RA, 0));
    else if (t == 1) good[1] = G1::pt_eq(pt_load<Fq>(sums + SC_KB1, 0), pt_load<Fq>(sums + SC_RB1, 0));
    else if (t == 2) good[2] = G2::pt_eq(pt_load<Fq2>(sums + SC_KB2, 0), pt_load<Fq2>(sums + SC_RB2, 0));
    else if (t == 3) a1[0] = G1::to_affine(pt_load<Fq>(sums + SC_KIC, 0));
    else if (t == 4) a1[1] = G1::to_affine(pt_load<Fq>(sums + SC_KL, 0));
    else if (t == 5) {
        G1::Pt r = pt_load<Fq>(sums + SC_RBE, 0);
        G1::add(r, pt_load<Fq>(sums + SC_RAL, 0));
        G1::add(r, pt_load<Fq>(sums + SC_RC, 0));
        a1[2] = G1::to_affine(G1::neg(r));
    } else if (t == 6) a1[3] = G1::to_affine(pt_load<Fq>(sums + SC_KH, 0));
    else if (t == 7) a1[4] = G1::to_affine(G1::neg(pt_load<Fq>(sums + SC_RH, 0)));
    else if (t == 8) a1[5] = aff_load<Fq>(g1, 0);                                  // delta_1
    else if (t == 9) { G1::Aff p = aff_load<Fq>(g1, 1); if (!G1::aff_is_inf(p)) p.y = Fq::neg(p.y); a1[6] = p; }   // -T_0
    // the G2 side of each pair: gamma_2, delta_2, U_0 | delta_2, U_0 | U_0, delta_2
    if (t < 7) a2[t] = aff_load<Fq2>(g2, t == 0 ? 0 : t == 1 || t == 3 || t == 6 ? 1 : 2);
    __syncthreads();
    if (t < 7) {
        fe12 r;
        miller_loop(r, !G1::aff_is_inf(a1[t]) && !G2::aff_is_inf(a2[t]), a1[t], a2[t], 0, nullptr, nullptr);
        f[t] = r;
    }
    __syncthreads();
    if (t < 3) {                                   // E4: pairs 0-2, E5: pairs 3-4, E6: pairs 5-6
        const int first = t == 0 ? 0 : t == 1 ? 3 : 5, last = t == 0 ? 3 : t == 1 ? 5 : 7;
        fe12 prod = f[first], e;
        for (int k = first + 1; k < last; k++) Fq12::mul(prod, prod, f[k]);
        Fq12::final_exponentiation(e, prod);
        good[3 + t] = Fq12::eq(e, Fq12::one()) ? 1u : 0u;
    }
    __syncthreads();
    if (t == 0) {
        uint32_t v = 0;
        for (int k = 5; k >= 0; k--) if (!good[k]) v = k + 1;
        *verdict = v;
    }
}

void setup_check_verdict(const void* sums, const void* g1, const void* g2, uint32_t* verdict, cudaStream_t st) {
    setup_check_verdict_kernel<<<1, 32, 0, st>>>((const uint8_t*)sums, (const uint8_t*)g1, (const uint8_t*)g2, verdict);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- delta update check
// b2g_delta_update_check: rec[i] = w_i after[i], rec[N + i] = w_i before[i] for the N = n_l + n_h points L || H of each key
// (G1 XYZZ); clears *ok when an after point has a coordinate >= p or lies off its curve
__global__ void __launch_bounds__(128) delta_weigh_kernel(const uint8_t* __restrict__ after, const uint8_t* __restrict__ before,
                                                          const uint32_t* __restrict__ w, uint32_t n, uint8_t* __restrict__ rec,
                                                          uint32_t* __restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool good = true;
    for (int k = 0; k < 2; k++) good &= fe_below_p(fe_load(after + ((size_t)i * 2 + k) * 32));
    const G1::Aff a = aff_load<Fq>(after, i), b = aff_load<Fq>(before, i);
    if (!good || !aff_on_curve<G1, Fq>(a)) atomicAnd(ok, 0u);
    uint32_t k[4];
    weight_load(k, w, i);
    pt_store<Fq>(rec, i, G1::mul_affine(a, k, 4));
    pt_store<Fq>(rec, (size_t)n + i, G1::mul_affine(b, k, 4));
}

// one block of 32 threads: threads 0-3 compute the four pairings e(d1', d2), e(d1, d2'), e(S', d2'), e(S, d2), thread 4
// checks the point rules, and thread 0 then gives the verdict.
// d = before d1 (64 B), before d2 (128 B), after d1, after d2; S' and S are the XYZZ sums at the first two tails.
__global__ void __launch_bounds__(32) delta_verdict_kernel(const uint8_t* __restrict__ d, const uint8_t* __restrict__ tails,
                                                           const uint32_t* __restrict__ ok, uint8_t* __restrict__ verdict) {
    __shared__ fe12 e[4];
    __shared__ uint32_t good;
    const uint32_t t = threadIdx.x;
    const G1::Aff d1 = aff_load<Fq>(d, 0), d1a = aff_load<Fq>(d + 192, 0);
    const G2::Aff d2 = aff_load<Fq2>(d + 64, 0), d2a = aff_load<Fq2>(d + 256, 0);
    if (t == 4) {
        bool g = *ok != 0;
        for (int k = 0; k < 6; k++) g &= fe_below_p(fe_load(d + 192 + 32 * k));
        g = g && aff_on_curve<G1, Fq>(d1a) && aff_on_curve<G2, Fq2>(d2a) && !G1::aff_is_inf(d1a) && !G2::aff_is_inf(d2a) &&
            !G2::aff_is_inf(d2) && g2_in_subgroup(d2a);
        good = g;
    } else if (t < 4) {
        G1::Aff p;
        if (t == 0) p = d1a;
        else if (t == 1) p = d1;
        else p = G1::to_affine(pt_load<Fq>(tails + (size_t)(t - 2) * TAIL_BYTES, 0));
        fe12 r;
        pairing(r, p, t == 0 || t == 3 ? d2 : d2a);
        e[t] = r;
    }
    __syncthreads();
    if (t == 0) *verdict = good && Fq12::eq(e[0], e[1]) && Fq12::eq(e[2], e[3]);
}

static void delta_check_run(b2g_ctx* ctx, const b2g_delta_key* a, const b2g_delta_key* b, const void* weights, uint8_t* verdict_out) {
    if (!ctx || !a || !b || !verdict_out) throw_error(B2G_E_SHAPE, "null pointer");
    if (!a->delta_g1 || !a->delta_g2 || !b->delta_g1 || !b->delta_g2 || (a->n_l && !a->l_query) || (a->n_h && !a->h_query) ||
        (b->n_l && !b->l_query) || (b->n_h && !b->h_query))
        throw_error(B2G_E_SHAPE, "null key buffer");
    const CtxView cv = ctx_idle(ctx);
    *verdict_out = 0;
    const uint64_t n64 = (uint64_t)a->n_l + a->n_h;
    if (n64 && !weights) throw_error(B2G_E_SHAPE, "null pointer");
    if (n64 >= (1ull << 31)) throw_error(B2G_E_DEVICE, "b2g_delta_update_check: more than 2^31 - 1 points");
    const uint32_t n = (uint32_t)n64;
    for (uint32_t i = 0; i < n; i++)
        if (all_zero((const uint8_t*)weights + 16 * (size_t)i, 16)) throw_error(B2G_E_INPUT, "weight " + std::to_string(i) + " is zero");
    if (a->n_l != b->n_l || a->n_h != b->n_h) return;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    // one allocation: the four delta points, after L || H, before L || H, the weights, 2n records, two scratch areas, the
    // tails of the two sums, the spans, the ok word and the verdict
    std::vector<Seg> segs(2);
    segs[0].first = 0; segs[0].count = n; segs[1].first = n; segs[1].count = n;
    std::vector<Span> spans;
    size_t scratch = 0;
    const std::vector<uint32_t> levels = n ? reduce_plan(segs, 128, spans, &scratch) : std::vector<uint32_t>();
    const size_t o_pts = 384, o_before = o_pts + (size_t)n * 64, o_w = o_before + (size_t)n * 64, o_rec = o_w + (size_t)n * 16;
    const size_t o_x = o_rec + (size_t)n * 256, o_y = o_x + std::max(scratch, (size_t)1) * 128;
    const size_t o_tails = (o_y + std::max(scratch, (size_t)1) * 128 + 255) & ~(size_t)255, o_spans = o_tails + 2 * TAIL_BYTES;
    const size_t o_ok = o_spans + std::max(spans.size(), (size_t)1) * sizeof(Span), bytes = o_ok + 8;
    DevArena mem(st);
    uint8_t* D = nullptr;
    try {
        D = mem.alloc(bytes);
    } catch (const B2gError&) {
        cudaGetLastError();
        throw_error(B2G_E_DEVICE, "b2g_delta_update_check: the device buffers (" + std::to_string((bytes + (1 << 20) - 1) >> 20) +
                                      " MiB) do not fit in device memory");
    }
    const uint32_t one = 1;
    CUDA_CHECK(cudaMemsetAsync(D + o_tails, 0, 2 * TAIL_BYTES, st));
    CUDA_CHECK(cudaMemcpyAsync(D + o_ok, &one, 4, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(D, a->delta_g1, 64, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(D + 64, a->delta_g2, 128, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(D + 192, b->delta_g1, 64, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(D + 256, b->delta_g2, 128, cudaMemcpyHostToDevice, st));
    if (n) {
        const size_t nl = a->n_l, nh = a->n_h;
        if (nl) CUDA_CHECK(cudaMemcpyAsync(D + o_pts, b->l_query, nl * 64, cudaMemcpyHostToDevice, st));
        if (nh) CUDA_CHECK(cudaMemcpyAsync(D + o_pts + nl * 64, b->h_query, nh * 64, cudaMemcpyHostToDevice, st));
        if (nl) CUDA_CHECK(cudaMemcpyAsync(D + o_before, a->l_query, nl * 64, cudaMemcpyHostToDevice, st));
        if (nh) CUDA_CHECK(cudaMemcpyAsync(D + o_before + nl * 64, a->h_query, nh * 64, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(D + o_w, weights, (size_t)n * 16, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(D + o_spans, spans.data(), spans.size() * sizeof(Span), cudaMemcpyHostToDevice, st));
        delta_weigh_kernel<<<(n + 127) / 128, 128, 0, st>>>(D + o_pts, D + o_before, (const uint32_t*)(D + o_w), n, D + o_rec,
                                                            (uint32_t*)(D + o_ok));
        g_launch_count += 1;
        reduce_run(levels, (const Span*)(D + o_spans), D + o_rec, 128, 128, nullptr, D + o_x, D + o_y,
                   [&](uint32_t blocks, const uint8_t* src, size_t stride, const Span* sp, const uint8_t* mask, uint8_t* dst) {
                       g1_sum_kernel<<<blocks, 128, 0, st>>>(src, stride, sp, mask, dst, D + o_tails);
                   });
    }
    delta_verdict_kernel<<<1, 32, 0, st>>>(D, D + o_tails, (const uint32_t*)(D + o_ok), D + o_ok + 4);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(verdict_out, D + o_ok + 4, 1, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

int setup_generators_check(const void* g1, const void* g2, cudaStream_t st) {
    if (!g1 && !g2) return 0;
    uint32_t* d_bad = nullptr;
    CUDA_CHECK(cudaMalloc(&d_bad, 2 * sizeof(uint32_t)));
    uint32_t bad[2] = {0, 0};
    cudaError_t e = cudaMemsetAsync(d_bad, 0, sizeof(bad), st);
    if (e == cudaSuccess) { setup_generators_kernel<<<1, 32, 0, st>>>(g1, g2, d_bad); g_launch_count += 1; e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpyAsync(bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d_bad);
    CUDA_CHECK(e);
    return bad[0] ? (int)bad[0] : (int)bad[1];
}

}  // namespace b2g

extern "C" {

int b2g_delta_update_check(b2g_ctx* ctx, const b2g_delta_key* before, const b2g_delta_key* after, const void* weights,
                           uint8_t* verdict_out) {
    return guarded([&] { delta_check_run(ctx, before, after, weights, verdict_out); });
}

int b2g_vk_load(b2g_ctx* ctx, const b2g_vk_desc* d, b2g_vk** out) {
    return guarded([&] { vk_load_many(ctx, 1, d, out, true); });
}

int b2g_vk_load_many(b2g_ctx* ctx, uint32_t n_keys, const b2g_vk_desc* descs, b2g_vk** out) {
    return guarded([&] { vk_load_many(ctx, n_keys, descs, out, false); });
}

int b2g_vk_free(b2g_vk* vk) {
    return guarded([&] {
        if (!vk) return;
        DevGuard g(vk->device);
        cudaDeviceSynchronize();
        delete vk;                                         // the last handle of a b2g_vk_load_many call frees its allocation
    });
}

int b2g_vk_alpha_beta(b2g_vk* vk, void* out) {
    return guarded([&] {
        if (!vk || !out) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(vk->device);
        CUDA_CHECK(cudaMemcpy(out, vk->d_eab, F12_BYTES, cudaMemcpyDeviceToHost));
    });
}

// the checks every call on a batch of proofs shares (pointers checked by the caller): count >= 1, no proof pending on the
// context; returns the context
static CtxView batch_args(const char* fn, b2g_ctx* ctx, uint32_t count) {
    if (count == 0) throw_error(B2G_E_SHAPE, std::string(fn) + ": count must be at least 1");
    const CtxView cv = ctx_idle(ctx);
    return cv;
}

// vbufs_ensure, reporting a batch that does not fit as B2G_E_DEVICE with advice
static void verify_bufs_ensure(const char* fn, VerifyBufs*& v, uint32_t count, size_t inputs, size_t parts, size_t batch = 0,
                               size_t comp = 0, size_t meta = 0) {
    try {
        vbufs_ensure(v, count, inputs, parts, batch, comp, meta);
    } catch (const B2gError& e) {
        if (e.code != B2G_E_DEVICE) throw;
        cudaGetLastError();
        throw_error(B2G_E_DEVICE, std::string(fn) + ": the device buffers of " + std::to_string(count) +
                                  " proofs do not fit in device memory; verify fewer per call (" + e.what() + ")");
    }
}

int b2g_proofs_decompress(b2g_ctx* ctx, uint32_t count, const void* compressed, uint8_t* proofs_out, uint8_t* ok_out) {
    return guarded([&] {
        if (!ctx || !compressed || !proofs_out || !ok_out) throw_error(B2G_E_SHAPE, "null pointer");
        const CtxView cv = batch_args("b2g_proofs_decompress", ctx, count);
        DevGuard g(cv.device);
        cudaStream_t st = cv.st;
        verify_bufs_ensure("b2g_proofs_decompress", *cv.vbufs, count, 0, 0, 0, comp_bytes(count));
        VerifyBufs& v = **cv.vbufs;
        const uint8_t* ok = decompress_enqueue(v, compressed, count, true, st);
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(proofs_out, v.d_proofs, (size_t)count * 256, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(ok_out, ok, count, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

int b2g_points_serialize(b2g_ctx* ctx, int g2, int compress, size_t n, const void* points_mont, void* out) {
    return guarded([&] {
        static const char* fn = "b2g_points_serialize";
        if (!ctx || !points_mont || !out) throw_error(B2G_E_SHAPE, std::string(fn) + ": null pointer");
        const size_t e = g2 ? 64 : 32;                     // bytes of one of x, y
        const uint64_t bad = points_slices(fn, ctx, n, 2 * e, compress ? e : 2 * e, points_mont, out,
            [&](const uint8_t* d_in, uint8_t* d_out, uint32_t m, uint64_t base, unsigned long long* d_bad, cudaStream_t st) {
                if (g2) points_serialize_kernel<Fq2><<<(m + 127) / 128, 128, 0, st>>>(d_in, m, compress, base, d_out, d_bad);
                else points_serialize_kernel<Fq><<<(m + 127) / 128, 128, 0, st>>>(d_in, m, compress, base, d_out, d_bad);
                g_launch_count += 1;
            });
        if (bad < n) throw_error(B2G_E_INPUT, std::string(fn) + ": point " + std::to_string(bad) + " has a coordinate >= p");
    });
}

int b2g_points_deserialize(b2g_ctx* ctx, int g2, int compress, size_t n, const void* in, void* points_out, uint64_t* first_bad_out) {
    return guarded([&] {
        static const char* fn = "b2g_points_deserialize";
        if (!ctx || !in || !points_out || !first_bad_out) throw_error(B2G_E_SHAPE, std::string(fn) + ": null pointer");
        const size_t e = g2 ? 64 : 32;
        *first_bad_out = points_slices(fn, ctx, n, compress ? e : 2 * e, 2 * e, in, points_out,
            [&](const uint8_t* d_in, uint8_t* d_out, uint32_t m, uint64_t base, unsigned long long* d_bad, cudaStream_t st) {
                const unsigned blocks = (m + 127) / 128;
                if (g2 && compress) points_deserialize_kernel<G2, Fq2, true><<<blocks, 128, 0, st>>>(d_in, m, base, d_out, d_bad);
                else if (g2) points_deserialize_kernel<G2, Fq2, false><<<blocks, 128, 0, st>>>(d_in, m, base, d_out, d_bad);
                else if (compress) points_deserialize_kernel<G1, Fq, true><<<blocks, 128, 0, st>>>(d_in, m, base, d_out, d_bad);
                else points_deserialize_kernel<G1, Fq, false><<<blocks, 128, 0, st>>>(d_in, m, base, d_out, d_bad);
                if (g2) points_g2_subgroup_kernel<<<blocks, 128, 0, st>>>(d_out, m, base, d_bad);
                g_launch_count += g2 ? 2 : 1;
            });
    });
}

int b2g_rerandomize_many(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* proofs, const void* r1_canon, const void* r2_canon,
                         uint8_t* proofs_out, uint8_t* ok_out) {
    return guarded([&] {
        static const char* fn = "b2g_rerandomize_many";
        if (!ctx || !vk || !proofs || !r1_canon || !r2_canon || !proofs_out || !ok_out) throw_error(B2G_E_SHAPE, "null pointer");
        const CtxView cv = batch_args(fn, ctx, count);
        if (vk->device != cv.device) throw_error(B2G_E_SHAPE, "the verifying key belongs to another device");
        DevGuard g(cv.device);
        cudaStream_t st = cv.st;
        // the buffers before the factors: a count whose buffers cannot fit is refused without reading count factors
        verify_bufs_ensure(fn, *cv.vbufs, count, 0, 0);
        VerifyBufs& v = **cv.vbufs;
        for (uint32_t i = 0; i < count; i++)
            for (const auto& [name, r] : {std::pair{"r1", r1_canon}, std::pair{"r2", r2_canon}}) {
                const uint32_t* k = (const uint32_t*)r + 8 * (size_t)i;
                if (all_zero(k, 32) || !below((const uint8_t*)k, R_WORDS))
                    throw_error(B2G_E_INPUT, std::string(fn) + ": factor " + name + " of proof " + std::to_string(i) +
                                             " is not in [1, r)");
            }
        // the factors and the output rows share the record area
        static_assert(REC_BYTES_V >= 2 * 32 + 256, "r1, r2 and the output row fit in a proof's record");
        uint8_t *d_r1 = v.d_rec, *d_r2 = v.d_rec + (size_t)count * 32, *d_out = v.d_rec + (size_t)count * 64;
        CUDA_CHECK(cudaMemcpyAsync(v.d_proofs, proofs, (size_t)count * 256, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(d_r1, r1_canon, (size_t)count * 32, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(d_r2, r2_canon, (size_t)count * 32, cudaMemcpyHostToDevice, st));
        rerandomize_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_proofs, d_r1, d_r2, vk->d_g2 + 2 * 128, count, d_out, v.d_verdict);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(proofs_out, d_out, (size_t)count * 256, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(ok_out, v.d_verdict, count, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

// the key record of a loaded key
static KeyRec key_rec(const b2g_vk* vk) {
    return {vk->d_lines, vk->d_eab, vk->d_tabs, vk->d_g1, vk->n_public, !vk->gamma_inf, !vk->delta_inf, 0};
}

// the device bytes of b2g_verify_many's tables for n_keys keys: the key records, then one segment per key
static size_t many_meta_bytes(size_t n_keys) { return n_keys * (sizeof(KeyRec) + sizeof(Seg)); }

// b2g_verify_many's uploads and four kernels on st, every proof under its own key: segment k holds the next counts[k]
// proofs, checked under vks[k] (counts[k] >= 1), and the public inputs of all proofs lie back to back.  On 256-byte rows, or
// on compressed rows decoded first (G2 check included); the verdicts go to v.d_verdict.  v.d_meta holds at least
// many_meta_bytes(vks.size()) bytes.
static void verify_many_enqueue(VerifyBufs& v, const std::vector<b2g_vk*>& vks, const std::vector<uint32_t>& counts,
                                const void* public_inputs, const void* proofs, bool compressed, cudaStream_t st) {
    const uint32_t n_segs = (uint32_t)vks.size();
    // the tables go up from a host buffer that outlives the call, as in batch_enqueue
    v.h_meta.assign(many_meta_bytes(n_segs), 0);
    KeyRec* keys = reinterpret_cast<KeyRec*>(v.h_meta.data());
    Seg* segs = reinterpret_cast<Seg*>(v.h_meta.data() + n_segs * sizeof(KeyRec));
    uint32_t count = 0;
    size_t inputs = 0;
    for (uint32_t k = 0; k < n_segs; k++) {
        keys[k] = key_rec(vks[k]);
        segs[k] = {inputs, k, count, counts[k], 0, 0, 0};
        count += counts[k]; inputs += (size_t)counts[k] * vks[k]->n_public;
    }
    const KeyRec* d_keys = reinterpret_cast<const KeyRec*>(v.d_meta);
    const Seg* d_segs = reinterpret_cast<const Seg*>(v.d_meta + n_segs * sizeof(KeyRec));
    CUDA_CHECK(cudaMemcpyAsync(v.d_meta, v.h_meta.data(), v.h_meta.size(), cudaMemcpyHostToDevice, st));
    if (compressed) decompress_enqueue(v, proofs, count, true, st);
    else CUDA_CHECK(cudaMemcpyAsync(v.d_proofs, proofs, (size_t)count * 256, cudaMemcpyHostToDevice, st));
    if (inputs) {
        CUDA_CHECK(cudaMemcpyAsync(v.d_pub, public_inputs, inputs * 32, cudaMemcpyHostToDevice, st));
        verify_inputs_kernel<<<(unsigned)((inputs + 3) / 4), 128, 0, st>>>(d_keys, d_segs, n_segs, (const uint32_t*)v.d_pub, inputs, v.d_part);
    }
    verify_prepare_kernel<<<(count + 127) / 128, 128, 0, st>>>(v.d_proofs, d_keys, d_segs, n_segs, v.d_part, count, v.d_rec);
    verify_miller_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_rec, d_keys, d_segs, n_segs, count, v.d_f);
    verify_final_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_rec, v.d_f, d_keys, d_segs, n_segs, count, v.d_verdict);
    g_launch_count += 3 + (inputs ? 1 : 0);
    CUDA_CHECK(cudaGetLastError());
}

// the device results of batch_enqueue: wf (one byte per proof: it parses and its B lies in G2) and one verdict per segment
struct BatchOut { const uint8_t* wf; const uint8_t* verdict; };

// the batch check over a segment table: segment g holds the next segs_in[g].count proofs, checked under vks[segs_in[g].key].
//   b2g_verify_batch         one segment, no mask; the verdict ANDs the ok word
//   b2g_verify_batch_locate  segments of LOCATE_GROUP proofs under one key, masked by wf
//   b2g_verify_batch_keys    one segment per key (keyed), no mask; each verdict ANDs its segment's ok byte
// on 256-byte rows or on compressed rows decoded on the context's stream before anything else reads them (batch_g2_kernel
// checks the decoded B, so the decoder skips the G2 check).  The results are ready once the context's stream is.
static BatchOut batch_enqueue(const char* fn, const CtxView& cv, const std::vector<b2g_vk*>& vks, const std::vector<SegIn>& segs_in,
                              bool masked, bool keyed, const void* public_inputs, const void* proofs, bool compressed,
                              const void* weights) {
    // the per-call tables: key records, segments, then the spans of the Miller-value products, of the r C sums and of the
    // prepared-input sums (one CTA per segment)
    std::vector<KeyRec> keys(vks.size());
    for (size_t k = 0; k < vks.size(); k++) keys[k] = key_rec(vks[k]);
    const uint32_t n_segs = (uint32_t)segs_in.size();
    std::vector<Seg> segs(n_segs);
    uint32_t count = 0, items = 0, n_pts_all = 0;
    size_t inputs = 0;
    for (uint32_t g = 0; g < n_segs; g++) {
        const SegIn& in = segs_in[g];
        const uint32_t n_public = keys[in.key].n_public, chunks = (in.count + SCALAR_CHUNK - 1) / SCALAR_CHUNK;
        segs[g] = {inputs, in.key, count, in.count, items, chunks, n_pts_all};
        count += in.count; inputs += (size_t)in.count * n_public; items += chunks * (n_public + 1); n_pts_all += n_public + 1;
    }
    std::vector<Span> spans;
    size_t lvl_f = 0, lvl_g = 0;
    const std::vector<uint32_t> levels_f = reduce_plan(segs, 64, spans, &lvl_f);
    const size_t sp_g = spans.size();
    const std::vector<uint32_t> levels_g = reduce_plan(segs, 128, spans, &lvl_g);
    const size_t sp_p = spans.size();
    for (uint32_t g = 0; g < n_segs; g++) spans.push_back({segs[g].pt, keys[segs_in[g].key].n_public + 1, TO_TAIL | g});
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t m_segs = up(keys.size() * sizeof(KeyRec)), m_spans = m_segs + up(segs.size() * sizeof(Seg));
    const size_t meta = m_spans + spans.size() * sizeof(Span);
    // scratch: weights, four reduction levels (x, y for the Miller values on the main stream, x2, y2 for the r C on side
    // stream 3; a segment of more than one CTA needs them), the chunk sums of the scalars, s_gj IC[j] per (segment, j), the
    // segment tails, wf, the segment verdicts, the segment ok bytes (keyed), two ok words (the one batch_prepare_kernel and
    // batch_g2_kernel clear, and one that stays set), the tables
    const size_t level = up(std::max(lvl_f * F12_BYTES, lvl_g * 128));
    const size_t o_w = 0, o_x = up((size_t)count * 16), o_y = o_x + level, o_x2 = o_y + level, o_y2 = o_x2 + level;
    const size_t o_part = o_y2 + level, o_pts = o_part + up((size_t)items * 32);
    const size_t o_tail = o_pts + up((size_t)n_pts_all * 128), o_wf = o_tail + (size_t)n_segs * TAIL_BYTES;
    const size_t o_gv = o_wf + up(count), o_sok = o_gv + up(n_segs), o_ok = o_sok + up(n_segs), o_meta = o_ok + 256;
    const size_t bytes = o_meta + up(meta);
    verify_bufs_ensure(fn, *cv.vbufs, count, inputs, 0, bytes, compressed ? comp_bytes(count) : 0);
    VerifyBufs& v = **cv.vbufs;
    batch_streams(v);
    // the tables go up in one copy from a host buffer that outlives the call
    v.h_meta.assign(meta, 0);
    memcpy(v.h_meta.data(), keys.data(), keys.size() * sizeof(KeyRec));
    memcpy(v.h_meta.data() + m_segs, segs.data(), segs.size() * sizeof(Seg));
    memcpy(v.h_meta.data() + m_spans, spans.data(), spans.size() * sizeof(Span));
    cudaStream_t st = cv.st, s2 = v.side[0], s3 = v.side[1];
    // ev_up: the uploads, before both side streams; ev_prep: the r C records, before side stream 3 sums them; ev_g2: wf,
    // before the masked product and r C sums (with a mask only); ev_pts: the prepared inputs, before the prepared pairs;
    // ev_s2, ev_s3: the end of each side stream, before the final kernel
    cudaEvent_t ev_up = v.ev[0], ev_prep = v.ev[1], ev_g2 = v.ev[2], ev_pts = v.ev[3], ev_s2 = v.ev[4], ev_s3 = v.ev[5];
    uint8_t* B = v.d_batch;
    uint8_t *tails = B + o_tail, *wf = B + o_wf, *gv = B + o_gv, *seg_ok = B + o_sok;
    const uint8_t* mask = masked ? wf : nullptr;
    const uint32_t* w = (const uint32_t*)(B + o_w);
    uint32_t* ok = (uint32_t*)(B + o_ok);
    const KeyRec* d_keys = (const KeyRec*)(B + o_meta);
    const Seg* d_segs = (const Seg*)(B + o_meta + m_segs);
    const Span* d_spans = (const Span*)(B + o_meta + m_spans);
    if (compressed) decompress_enqueue(v, proofs, count, false, st);
    else CUDA_CHECK(cudaMemcpyAsync(v.d_proofs, proofs, (size_t)count * 256, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(B + o_w, weights, (size_t)count * 16, cudaMemcpyHostToDevice, st));
    if (inputs) CUDA_CHECK(cudaMemcpyAsync(v.d_pub, public_inputs, inputs * 32, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(B + o_meta, v.h_meta.data(), meta, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemsetAsync(ok, 0xff, 8, st));
    if (keyed) CUDA_CHECK(cudaMemsetAsync(seg_ok, 1, n_segs, st));
    CUDA_CHECK(cudaMemsetAsync(v.d_rec, 0, (size_t)count * REC_BYTES_V, st));
    CUDA_CHECK(cudaEventRecord(ev_up, st));
    // main stream: per-proof parse and scaling, then the Miller values.  With one verdict for the batch the Miller kernel
    // reads the ok word and skips a batch that has already failed; with a verdict per segment, every proof needs its Miller
    // value, so it reads the word that stays set.
    batch_prepare_kernel<<<(count + 127) / 128, 128, 0, st>>>(v.d_proofs, w, count, v.d_rec, ok);
    CUDA_CHECK(cudaEventRecord(ev_prep, st));
    batch_miller_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_rec, masked || keyed ? ok + 1 : ok, count, v.d_f);
    // side stream 2: the segment scalars and prepared inputs, e(alpha, beta)^s_g0, and the G2 membership of every B: first
    // when wf masks the sums, last when only the verdicts need it (keyed: then the segment ok bytes)
    auto g2 = [&] {
        batch_g2_kernel<<<(count + 127) / 128, 128, 0, s2>>>(v.d_proofs, count, wf, ok);
        CUDA_CHECK(cudaEventRecord(ev_g2, s2));
    };
    CUDA_CHECK(cudaStreamWaitEvent(s2, ev_up, 0));
    if (masked) g2();
    batch_scalars_kernel<<<items, 128, 0, s2>>>(w, (const uint32_t*)v.d_pub, mask, d_segs, n_segs, d_keys, B + o_part);
    batch_inputs_kernel<<<(n_pts_all + 3) / 4, 128, 0, s2>>>(B + o_part, d_segs, n_segs, d_keys, n_pts_all, B + o_pts, tails);
    g1_sum_kernel<<<n_segs, 128, 0, s2>>>(B + o_pts, 128, d_spans + sp_p, nullptr, nullptr, tails + TAIL_PREP);
    CUDA_CHECK(cudaEventRecord(ev_pts, s2));
    batch_rhs_kernel<<<(n_segs + 63) / 64, 64, 0, s2>>>(tails, n_segs, d_segs, d_keys);
    if (!masked) g2();
    if (keyed) batch_segment_ok_kernel<<<(count + 127) / 128, 128, 0, s2>>>(wf, d_segs, n_segs, count, seg_ok);
    CUDA_CHECK(cudaEventRecord(ev_s2, s2));
    // side stream 3, once the r C (and wf, with a mask) exist: the segment sums of r C, then, once the prepared inputs exist,
    // the segments' prepared pairs
    CUDA_CHECK(cudaStreamWaitEvent(s3, ev_prep, 0));
    if (masked) CUDA_CHECK(cudaStreamWaitEvent(s3, ev_g2, 0));
    reduce_run(levels_g, d_spans + sp_g, v.d_rec + BREC_RC, REC_BYTES_V, 128, mask, B + o_x2, B + o_y2,
               [&](uint32_t blocks, const uint8_t* src, size_t stride, const Span* sp, const uint8_t* m, uint8_t* dst) {
                   g1_sum_kernel<<<blocks, 128, 0, s3>>>(src, stride, sp, m, dst, tails + TAIL_RC);
               });
    CUDA_CHECK(cudaStreamWaitEvent(s3, ev_pts, 0));
    batch_pairs_kernel<<<(n_segs + 63) / 64, 64, 0, s3>>>(tails, n_segs, d_segs, d_keys);
    CUDA_CHECK(cudaEventRecord(ev_s3, s3));
    // main stream: the segment products of the Miller values, then the segment verdicts
    if (masked) CUDA_CHECK(cudaStreamWaitEvent(st, ev_g2, 0));
    reduce_run(levels_f, d_spans, v.d_f, F12_BYTES, F12_BYTES, mask, B + o_x, B + o_y,
               [&](uint32_t blocks, const uint8_t* src, size_t stride, const Span* sp, const uint8_t* m, uint8_t* dst) {
                   f12_product_kernel<<<blocks, 64, 0, st>>>(src, stride, sp, m, dst, tails + TAIL_F);
               });
    CUDA_CHECK(cudaStreamWaitEvent(st, ev_s2, 0));
    CUDA_CHECK(cudaStreamWaitEvent(st, ev_s3, 0));
    batch_final_kernel<<<(n_segs + 63) / 64, 64, 0, st>>>(tails, n_segs, masked || keyed ? nullptr : ok, keyed ? seg_ok : nullptr, gv);
    g_launch_count += keyed ? 10 : 9;
    CUDA_CHECK(cudaGetLastError());
    return {wf, gv};
}

// key batches as one run of proofs: one entry per batch that holds proofs (vks, counts, and its index among the caller's
// batches in `at`), and their proofs, public inputs and weights back to back.  With one such batch these are the caller's
// arrays; with more they are packed into one host array each, so that each goes up in one copy.
struct KeysPacked {
    std::vector<b2g_vk*> vks;
    std::vector<uint32_t> counts, at;
    uint32_t total = 0;
    size_t inputs = 0;
    const void *proofs = nullptr, *public_inputs = nullptr, *weights = nullptr;
    std::vector<uint8_t> rows_h, pubs_h, ws_h;
};

// the shape checks of a one-key verifier (b2g_verify_many, b2g_verify_batch, b2g_verify_batch_locate and their compressed
// forms) on the key batch made of its arguments, the weights only when its kind takes them; returns the number of proofs
static uint32_t one_key_shape(b2g_ctx* ctx, const b2g_key_batch& b, bool weighted, const uint8_t* verdicts_out) {
    if (!ctx || !b.vk || !b.proofs || !verdicts_out || (weighted && !b.weights) || (b.vk->n_public && !b.public_inputs))
        throw_error(B2G_E_SHAPE, "null pointer");
    return b.count;
}

// the shape checks of a key-table verifier (b2g_verify_batch_keys, b2g_verify_batch_keys_locate and their compressed forms),
// each message about a row naming the key index; returns the number of proofs
static uint32_t keys_shape(const char* fn, b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, const uint8_t* verdicts_out) {
    if (!ctx || !batches || !verdicts_out) throw_error(B2G_E_SHAPE, "null pointer");
    if (n_keys == 0) throw_error(B2G_E_SHAPE, std::string(fn) + ": n_keys must be at least 1");
    auto at = [&](uint32_t k) { return std::string(fn) + ": key " + std::to_string(k) + ": "; };
    uint64_t total = 0;
    for (uint32_t k = 0; k < n_keys; k++) {
        const b2g_key_batch& b = batches[k];
        if (!b.vk) throw_error(B2G_E_SHAPE, at(k) + "null verifying key");
        if (b.count && (!b.proofs || !b.weights || (b.vk->n_public && !b.public_inputs))) throw_error(B2G_E_SHAPE, at(k) + "null pointer");
        total += b.count;
    }
    if (total == 0) throw_error(B2G_E_SHAPE, std::string(fn) + ": every key batch is empty; at least one proof is needed");
    if (total > UINT32_MAX) throw_error(B2G_E_SHAPE, std::string(fn) + ": more than 2^32 - 1 proofs in all");
    return (uint32_t)total;
}

// the content checks of one key batch, for every verifier: its key lies on the context's device, every public input is
// below r and, when the kind takes weights, no weight is zero.  In a key table (key >= 0) each message names the key index.
static void batch_check(const char* fn, int64_t key, const CtxView& cv, const b2g_key_batch& b, bool weighted) {
    auto fail = [&](int code, const std::string& what) {
        throw_error(code, key < 0 ? what : std::string(fn) + ": key " + std::to_string(key) + ": " + what);
    };
    if (b.vk->device != cv.device) fail(B2G_E_SHAPE, "the verifying key belongs to another device");
    const uint32_t n_public = b.vk->n_public;
    const uint32_t* pub = (const uint32_t*)b.public_inputs;
    for (size_t i = 0; i < (size_t)b.count * n_public; i++)
        if (!below((const uint8_t*)(pub + 8 * i), R_WORDS)) fail(B2G_E_INPUT, "public input " + std::to_string(i % n_public) + " of proof " + std::to_string(i / n_public) +
                                                     " is not below the scalar field modulus r");
    for (uint32_t i = 0; weighted && i < b.count; i++)
        if (all_zero((const uint8_t*)b.weights + 16 * (size_t)i, 16)) fail(B2G_E_INPUT, "weight " + std::to_string(i) + " is zero");
}

// the key batches (checked) as one run of proofs
static KeysPacked keys_pack(uint32_t n_keys, const b2g_key_batch* batches, bool compressed) {
    uint32_t used = 0, last = 0;
    for (uint32_t k = 0; k < n_keys; k++) if (batches[k].count) { used++; last = k; }
    KeysPacked p;
    if (used == 1) {
        const b2g_key_batch& b = batches[last];
        p.vks = {b.vk}; p.counts = {b.count}; p.at = {last};
        p.total = b.count; p.inputs = (size_t)b.count * b.vk->n_public;
        p.proofs = b.proofs; p.public_inputs = b.public_inputs; p.weights = b.weights;
        return p;
    }
    for (uint32_t k = 0; k < n_keys; k++) {
        p.total += batches[k].count;
        p.inputs += (size_t)batches[k].count * batches[k].vk->n_public;
    }
    const size_t row = compressed ? COMP_BYTES : 256;
    p.rows_h.resize((size_t)p.total * row); p.pubs_h.resize(p.inputs * 32); p.ws_h.resize((size_t)p.total * 16);
    size_t n = 0, x = 0;
    for (uint32_t k = 0; k < n_keys; k++) {
        const b2g_key_batch& b = batches[k];
        if (!b.count) continue;
        const size_t nx = (size_t)b.count * b.vk->n_public * 32;
        memcpy(p.rows_h.data() + n * row, b.proofs, b.count * row);
        memcpy(p.ws_h.data() + n * 16, b.weights, (size_t)b.count * 16);
        if (nx) memcpy(p.pubs_h.data() + x, b.public_inputs, nx);
        p.vks.push_back(b.vk); p.counts.push_back(b.count); p.at.push_back(k);
        n += b.count; x += nx;
    }
    p.proofs = p.rows_h.data(); p.public_inputs = p.pubs_h.data(); p.weights = p.ws_h.data();
    return p;
}

// the per-proof verdicts of b2g_verify_batch_locate and b2g_verify_batch_keys_locate, p.total bytes in p's order.  The batch
// check runs once per segment of at most LOCATE_GROUP consecutive proofs of one key (a key's segments start at its first
// proof), masked by wf; the well-formed proofs of the segments that fail it then go through b2g_verify_many's kernels in one
// pass, each under its own key, compacted on the host from p's rows.
static void locate_run(const char* fn, const CtxView& cv, const KeysPacked& p, bool compressed, uint8_t* verdicts_out) {
    cudaStream_t st = cv.st;
    std::vector<SegIn> segs;
    for (uint32_t k = 0; k < (uint32_t)p.vks.size(); k++)
        for (uint32_t f = 0; f < p.counts[k]; f += LOCATE_GROUP) segs.push_back({k, std::min(LOCATE_GROUP, p.counts[k] - f)});
    const BatchOut r = batch_enqueue(fn, cv, p.vks, segs, true, false, p.public_inputs, p.proofs, compressed, p.weights);
    std::vector<uint8_t> ok_h(p.total), gv_h(segs.size());
    CUDA_CHECK(cudaMemcpyAsync(ok_h.data(), r.wf, p.total, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(gv_h.data(), r.verdict, segs.size(), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    // the verdicts: 0 for a malformed proof, 1 in a segment that holds, else b2g_verify_many's verdict.  The proofs checked
    // again (idx, with their first public-input scalar in xs) keep the keys' order: one b2g_verify_many segment per key
    // among them (vks2, counts2).
    std::vector<uint8_t> out(p.total);
    std::vector<uint32_t> idx, counts2;
    std::vector<size_t> xs;
    std::vector<b2g_vk*> vks2;
    uint32_t i = 0, prev = UINT32_MAX;
    size_t x = 0, inputs2 = 0;
    for (uint32_t g = 0; g < (uint32_t)segs.size(); g++) {
        const uint32_t key = segs[g].key, n_public = p.vks[key]->n_public;
        for (uint32_t t = 0; t < segs[g].count; t++, i++, x += n_public) {
            out[i] = ok_h[i] && gv_h[g];
            if (!ok_h[i] || gv_h[g]) continue;
            if (key != prev) { vks2.push_back(p.vks[key]); counts2.push_back(0); prev = key; }
            counts2.back()++;
            idx.push_back(i); xs.push_back(x); inputs2 += n_public;
        }
    }
    if (!idx.empty()) {
        // when every proof is checked again, p's rows are already the compact ones
        const uint32_t m = (uint32_t)idx.size();
        const bool whole = m == p.total;
        const size_t row = compressed ? COMP_BYTES : 256;
        std::vector<uint8_t> rows(whole ? 0 : (size_t)m * row), pubs(whole ? 0 : inputs2 * 32), many(m);
        size_t y = 0;
        for (uint32_t k = 0, s = 0, in_s = 0; k < m && !whole; k++) {            // proof k is the in_s-th of segment s
            memcpy(rows.data() + (size_t)k * row, (const uint8_t*)p.proofs + (size_t)idx[k] * row, row);
            const size_t pub_row = (size_t)vks2[s]->n_public * 32;
            if (pub_row) memcpy(pubs.data() + y, (const uint8_t*)p.public_inputs + xs[k] * 32, pub_row);
            y += pub_row;
            if (++in_s == counts2[s]) { s++; in_s = 0; }
        }
        verify_bufs_ensure(fn, *cv.vbufs, p.total, p.inputs, inputs2, 0, compressed ? comp_bytes(p.total) : 0, many_meta_bytes(vks2.size()));
        verify_many_enqueue(**cv.vbufs, vks2, counts2, whole ? p.public_inputs : pubs.data(), whole ? p.proofs : rows.data(), compressed, st);
        CUDA_CHECK(cudaMemcpyAsync(many.data(), (*cv.vbufs)->d_verdict, m, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        for (uint32_t k = 0; k < m; k++) out[idx[k]] = many[k];
    }
    memcpy(verdicts_out, out.data(), p.total);
}

// how a verifier call runs its key batches:
//   VERIFY_MANY    b2g_verify_many's kernels, one verdict per proof
//   VERIFY_BATCH   the batch check with one segment, unmasked: b2g_verify_batch's one verdict
//   VERIFY_KEYS    the batch check with one segment per key batch that holds proofs (keyed): one verdict per key batch
//   VERIFY_LOCATE  locate_run, one verdict per proof
// VERIFY_BATCH stays apart from VERIFY_KEYS on one key: it has one launch fewer, and its Miller kernel skips a batch that
// has already failed.
enum VerifyKind { VERIFY_MANY, VERIFY_BATCH, VERIFY_KEYS, VERIFY_LOCATE };

// every verifier on 256-byte rows, or on compressed rows: the checks, then kind's run over the key batches, whose verdicts
// go to verdicts_out (a key batch without proofs gets 1 under VERIFY_KEYS, and none under VERIFY_LOCATE).  `table`: the
// batches are the caller's key table, not the one batch made of a one-key verifier's arguments.
static void verify_run(const char* fn, b2g_ctx* ctx, VerifyKind kind, bool table, uint32_t n_keys, const b2g_key_batch* batches,
                       bool compressed, uint8_t* verdicts_out) {
    const bool weighted = kind != VERIFY_MANY;
    const uint32_t total = table ? keys_shape(fn, ctx, n_keys, batches, verdicts_out) : one_key_shape(ctx, batches[0], weighted, verdicts_out);
    const CtxView cv = batch_args(fn, ctx, total);
    for (uint32_t k = 0; k < n_keys; k++) batch_check(fn, table ? (int64_t)k : -1, cv, batches[k], weighted);
    const KeysPacked p = keys_pack(n_keys, batches, compressed);
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    if (kind == VERIFY_LOCATE) {
        locate_run(fn, cv, p, compressed, verdicts_out);
    } else if (kind == VERIFY_MANY) {
        verify_bufs_ensure(fn, *cv.vbufs, p.total, p.inputs, p.inputs, 0, compressed ? comp_bytes(p.total) : 0, many_meta_bytes(p.vks.size()));
        verify_many_enqueue(**cv.vbufs, p.vks, p.counts, p.public_inputs, p.proofs, compressed, st);
        CUDA_CHECK(cudaMemcpyAsync(verdicts_out, (*cv.vbufs)->d_verdict, p.total, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    } else {
        std::vector<SegIn> segs;
        for (uint32_t k = 0; k < (uint32_t)p.vks.size(); k++) segs.push_back({k, p.counts[k]});
        const BatchOut r = batch_enqueue(fn, cv, p.vks, segs, false, kind == VERIFY_KEYS, p.public_inputs, p.proofs, compressed, p.weights);
        std::vector<uint8_t> gv(segs.size());
        CUDA_CHECK(cudaMemcpyAsync(gv.data(), r.verdict, segs.size(), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        std::fill(verdicts_out, verdicts_out + n_keys, 1);
        for (size_t k = 0; k < segs.size(); k++) verdicts_out[p.at[k]] = gv[k];
    }
}

int b2g_verify_many(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs, uint8_t* verdicts_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, proofs, nullptr};
    return guarded([&] { verify_run("b2g_verify_many", ctx, VERIFY_MANY, false, 1, &b, false, verdicts_out); });
}

int b2g_verify_many_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* compressed,
                               uint8_t* verdicts_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, compressed, nullptr};
    return guarded([&] { verify_run("b2g_verify_many_compressed", ctx, VERIFY_MANY, false, 1, &b, true, verdicts_out); });
}

int b2g_verify_batch(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs, const void* weights,
                     uint8_t* verdict_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, proofs, weights};
    return guarded([&] { verify_run("b2g_verify_batch", ctx, VERIFY_BATCH, false, 1, &b, false, verdict_out); });
}

int b2g_verify_batch_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* compressed,
                                const void* weights, uint8_t* verdict_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, compressed, weights};
    return guarded([&] { verify_run("b2g_verify_batch_compressed", ctx, VERIFY_BATCH, false, 1, &b, true, verdict_out); });
}

int b2g_verify_batch_locate(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs, const void* weights,
                            uint8_t* verdicts_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, proofs, weights};
    return guarded([&] { verify_run("b2g_verify_batch_locate", ctx, VERIFY_LOCATE, false, 1, &b, false, verdicts_out); });
}

int b2g_verify_batch_locate_compressed(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* compressed,
                                       const void* weights, uint8_t* verdicts_out) {
    const b2g_key_batch b = {vk, count, 0, public_inputs, compressed, weights};
    return guarded([&] { verify_run("b2g_verify_batch_locate_compressed", ctx, VERIFY_LOCATE, false, 1, &b, true, verdicts_out); });
}

int b2g_verify_batch_keys(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out) {
    return guarded([&] { verify_run("b2g_verify_batch_keys", ctx, VERIFY_KEYS, true, n_keys, batches, false, verdicts_out); });
}

int b2g_verify_batch_keys_compressed(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out) {
    return guarded([&] { verify_run("b2g_verify_batch_keys_compressed", ctx, VERIFY_KEYS, true, n_keys, batches, true, verdicts_out); });
}

int b2g_verify_batch_keys_locate(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out) {
    return guarded([&] { verify_run("b2g_verify_batch_keys_locate", ctx, VERIFY_LOCATE, true, n_keys, batches, false, verdicts_out); });
}

int b2g_verify_batch_keys_locate_compressed(b2g_ctx* ctx, uint32_t n_keys, const b2g_key_batch* batches, uint8_t* verdicts_out) {
    return guarded([&] {
        verify_run("b2g_verify_batch_keys_locate_compressed", ctx, VERIFY_LOCATE, true, n_keys, batches, true, verdicts_out);
    });
}

}  // extern "C"
