// contribute.cu - b2g_points_scale, a variable-base product per point with one scalar per point, and b2g_powers_contribute, the
// phase-1 contribution (`snarkjs powersoftau contribute`) it serves.
//
//   split      G1 (GLV): k = k1 + k2 lambda (mod r), |k1|, |k2| < 2^128, by Babai rounding on a short basis (A1, B1), (A2, B2):
//              c1 = (k G1R) >> 256, c2 = (k G2R) >> 256, k1 = k - c1 A1 - c2 A2, k2 = -c1 B1 - c2 B2 in two's complement mod
//              2^192; phi(x, y) = (beta x, y) acts as [lambda].  G2 (GLS): psi, the twist Frobenius, acts on G2 as [6x^2]
//              (p = r + 6x^2), so k1 = k mod 6x^2, k2 = k div 6x^2 < 2^127: a quotient estimate (k MU) >> 256, MU =
//              floor(2^256 / 6x^2), then at most a few subtractions.  The constants are derived in tests/ptau_contribute_model.py.
//   windows    each half h < 2^128 is read as 33 signed digits d_i = nib_i(h) + bit_(4i-1)(h) - 16 bit_(4i+3)(h) in [-8, 8],
//              h = sum d_i 16^i, from the top and without storage: the carry into digit i is bit 4i - 1.  Every lane runs the
//              same schedule: per digit 4 doublings, then one addition per half of +-T[|d| - 1] (the second half through the
//              endomorphism, applied to the loaded entry), T[j] = (j + 1) P in XYZZ in a per-thread table.  A digit only selects
//              the entry and its sign; a zero digit adds nothing.  The exceptional additions (equal or opposite points) are
//              add's, so the result is exact for every scalar.
//   streaming  slices of POWERS_SLICE points: a host copy into one of two pinned buffers, an asynchronous copy to the device on
//              a copy stream, the products in place, the copy back into the same pinned buffer on the context's stream, and the
//              host copy of slice k to its output after slice k + 1 has been queued.
#include <algorithm>
#include <cstring>
#include <string>
#include "../../include/b2groth.h"
#include "ec.cuh"
#include "fixed.cuh"
#include "msm.cuh"
#include "setup.cuh"
#include "stage.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {

// little-endian 32-bit words of the split constants (tests/ptau_contribute_model.py checks them against the model)
__constant__ uint32_t SPLIT_BETA[8] = {0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du};
__constant__ uint32_t SPLIT_A1[2] = {0x94d213e3u, 0x89d32568u};                               // = B2
__constant__ uint32_t SPLIT_B1[4] = {0x7d4f1128u, 0x8211bbebu, 0xeeb859fcu, 0x6f4d8248u};     // -B1 (B1 < 0)
__constant__ uint32_t SPLIT_A2[4] = {0x1221250bu, 0x0be4e154u, 0xeeb859fdu, 0x6f4d8248u};
__constant__ uint32_t SPLIT_G1R[3] = {0xc7e0b3d7u, 0xd91d232eu, 0x00000002u};
__constant__ uint32_t SPLIT_G2R[5] = {0x391eb18eu, 0x7a7bd9d4u, 0xa773d2cfu, 0x4ccef014u, 0x00000002u};
__constant__ uint32_t SPLIT_D[4] = {0xe87cfd46u, 0xf83e9682u, 0xeeb859fbu, 0x6f4d8248u};      // 6x^2
__constant__ uint32_t SPLIT_MU[5] = {0xc8e01941u, 0x2cb62031u, 0xa773d2d5u, 0x4ccef014u, 0x00000002u};

constexpr int SCALE_DIGITS = 33;                         // signed 4-bit digits of a half below 2^128

// the low NO words of a (NA words) times b (NB words)
template <int NA, int NB, int NO>
__device__ __forceinline__ void mp_mul(const uint32_t* a, const uint32_t* b, uint32_t* o) {
    #pragma unroll
    for (int i = 0; i < NO; i++) o[i] = 0;
    #pragma unroll
    for (int i = 0; i < NA; i++) {
        uint64_t carry = 0;
        #pragma unroll
        for (int j = 0; j < NB; j++) {
            if (i + j < NO) {
                const uint64_t t = (uint64_t)a[i] * b[j] + o[i + j] + carry;
                o[i + j] = (uint32_t)t;
                carry = t >> 32;
            }
        }
        if (i + NB < NO) o[i + NB] = (uint32_t)carry;
    }
}

// a -= b (N words, mod 2^(32 N)); b has NB <= N words
template <int N, int NB>
__device__ __forceinline__ void mp_sub(uint32_t* a, const uint32_t* b) {
    uint32_t borrow = 0;
    #pragma unroll
    for (int i = 0; i < N; i++) {
        const uint64_t t = (uint64_t)a[i] - (i < NB ? b[i] : 0u) - borrow;
        a[i] = (uint32_t)t;
        borrow = (uint32_t)(t >> 63);
    }
}

// a = -a (N words, two's complement)
template <int N>
__device__ __forceinline__ void mp_neg(uint32_t* a) {
    uint32_t carry = 1;
    #pragma unroll
    for (int i = 0; i < N; i++) {
        const uint64_t t = (uint64_t)(~a[i]) + carry;
        a[i] = (uint32_t)t;
        carry = (uint32_t)(t >> 32);
    }
}

// the two halves of a split: magnitudes below 2^128 and their signs
struct Split { uint32_t h[2][4]; bool neg[2]; };

// k = k1 + k2 lambda (mod r) for a canonical k < r
__device__ __forceinline__ Split glv_split(const uint32_t* k) {
    uint32_t p1[11], p2[13], c1[3], c2[5], t[6], k1[6], k2[6];
    mp_mul<8, 3, 11>(k, SPLIT_G1R, p1);
    mp_mul<8, 5, 13>(k, SPLIT_G2R, p2);
    #pragma unroll
    for (int i = 0; i < 3; i++) c1[i] = p1[8 + i];
    #pragma unroll
    for (int i = 0; i < 5; i++) c2[i] = p2[8 + i];
    #pragma unroll
    for (int i = 0; i < 6; i++) k1[i] = k[i];
    mp_mul<3, 2, 6>(c1, SPLIT_A1, t);
    mp_sub<6, 6>(k1, t);
    mp_mul<5, 4, 6>(c2, SPLIT_A2, t);
    mp_sub<6, 6>(k1, t);
    mp_mul<3, 4, 6>(c1, SPLIT_B1, k2);                   // c1 (-B1)
    mp_mul<5, 2, 6>(c2, SPLIT_A1, t);                    // c2 B2, B2 = A1
    mp_sub<6, 6>(k2, t);
    Split s;
    s.neg[0] = k1[5] >> 31;
    s.neg[1] = k2[5] >> 31;
    if (s.neg[0]) mp_neg<6>(k1);
    if (s.neg[1]) mp_neg<6>(k2);
    #pragma unroll
    for (int i = 0; i < 4; i++) { s.h[0][i] = k1[i]; s.h[1][i] = k2[i]; }
    return s;
}

// k = k1 + k2 6x^2 with k1 = k mod 6x^2, for a canonical k < r
__device__ __forceinline__ Split gls_split(const uint32_t* k) {
    uint32_t p[13], q[5], t[5], rem[5];
    mp_mul<8, 5, 13>(k, SPLIT_MU, p);
    #pragma unroll
    for (int i = 0; i < 5; i++) { q[i] = p[8 + i]; rem[i] = k[i]; }
    mp_mul<5, 4, 5>(q, SPLIT_D, t);
    mp_sub<5, 5>(rem, t);
    // the estimate is at most a few below the quotient: while rem >= 6x^2, subtract it and count
    for (;;) {
        bool ge = rem[4] != 0;
        if (!ge) {
            ge = true;
            for (int i = 3; i >= 0; i--)
                if (rem[i] != SPLIT_D[i]) { ge = rem[i] > SPLIT_D[i]; break; }
        }
        if (!ge) break;
        mp_sub<5, 4>(rem, SPLIT_D);
        const uint32_t one[1] = {1u};
        mp_neg<5>(q); mp_sub<5, 1>(q, one); mp_neg<5>(q);   // q += 1
    }
    Split s;
    s.neg[0] = s.neg[1] = false;
    #pragma unroll
    for (int i = 0; i < 4; i++) { s.h[0][i] = rem[i]; s.h[1][i] = q[i]; }
    return s;
}

__device__ __forceinline__ uint32_t half_word(const uint32_t* h, int w) {
    return w == 0 ? h[0] : w == 1 ? h[1] : w == 2 ? h[2] : w == 3 ? h[3] : 0u;
}

// digit i of a half: nib_i + bit (4i - 1) - 16 bit (4i + 3), in [-8, 8]
__device__ __forceinline__ int half_digit(const uint32_t* h, int i) {
    const int b = 4 * i;
    const uint32_t nib = (half_word(h, b >> 5) >> (b & 31)) & 15u;
    const uint32_t lo = b ? (half_word(h, (b - 1) >> 5) >> ((b - 1) & 31)) & 1u : 0u;
    return (int)(nib + lo) - (int)((nib >> 3) << 4);
}

template <class C> struct Endo;
template <> struct Endo<G1> {            // phi(x, y) = (beta x, y): on XYZZ, X beta
    static __device__ __forceinline__ G1::Pt apply(const G1::Pt& p) {
        G1::Pt r = p;
        fe b; for (int i = 0; i < 8; i++) b.l[i] = SPLIT_BETA[i];
        r.x = Fq::mul(p.x, b);
        return r;
    }
    static __device__ __forceinline__ Split split(const uint32_t* k) { return glv_split(k); }
};
template <> struct Endo<G2> {            // psi, the twist Frobenius
    static __device__ __forceinline__ G2::Pt apply(const G2::Pt& p) {
        G2::Pt r;
        r.x = Fq2::mul(conj(p.x), psi_coeff(0));
        r.y = Fq2::mul(conj(p.y), psi_coeff(1));
        r.zz = conj(p.zz);
        r.zzz = conj(p.zzz);
        return r;
    }
    static __device__ __forceinline__ fe2 conj(const fe2& a) { fe2 r; r.c0 = a.c0; r.c1 = Fq::neg(a.c1); return r; }
    static __device__ __forceinline__ fe2 psi_coeff(int y);
    static __device__ __forceinline__ Split split(const uint32_t* k) { return gls_split(k); }
};

// xi^((p - 1) / 3) and xi^((p - 1) / 2), Montgomery (c0, c1): psi(x, y) = (conj(x) PSI_X, conj(y) PSI_Y)
__constant__ uint32_t SPLIT_PSI[2][16] = {
    {0x4563ab30u, 0xb5773b10u, 0xa9aa6454u, 0x347f91c8u, 0x242e0991u, 0x7a007127u, 0x118214ecu, 0x1956bcd8u,
     0xa0aa4757u, 0x6e849f1eu, 0x89f89141u, 0xaa1c7b6du, 0xfae0ca3au, 0xb6e713cdu, 0x4e82ebc3u, 0x26694fbbu},
    {0x2936b629u, 0xe4bbdd0cu, 0xe133bacbu, 0xbb30f162u, 0xf9645366u, 0x31a9d1b6u, 0xa500f8ddu, 0x253570beu,
     0x5ffe77c7u, 0xa1d77ce4u, 0x7826d1dbu, 0x07affd11u, 0xbb7edc6bu, 0x6d16bd27u, 0x85defeccu, 0x2c872002u}};
__device__ __forceinline__ fe2 Endo<G2>::psi_coeff(int y) {
    fe2 r;
    for (int i = 0; i < 8; i++) { r.c0.l[i] = SPLIT_PSI[y][i]; r.c1.l[i] = SPLIT_PSI[y][8 + i]; }
    return r;
}

// k P for an affine P and a canonical k < r: the split, the table T[j] = (j + 1) P, and 33 lane-uniform signed windows
template <class C>
__device__ __forceinline__ typename C::Pt scale_point(const typename C::Aff& p, const uint32_t* k) {
    using Pt = typename C::Pt;
    Pt tab[8];
    tab[0] = C::from_affine(p);
    tab[1] = C::dbl_affine(p);
    #pragma unroll 1
    for (int j = 2; j < 8; j++) { tab[j] = tab[j - 1]; C::madd(tab[j], p); }
    const Split s = Endo<C>::split(k);
    Pt acc = C::infinity();
    #pragma unroll 1
    for (int i = SCALE_DIGITS - 1; i >= 0; i--) {
        #pragma unroll
        for (int d = 0; d < 4; d++) acc = C::dbl(acc);
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            const int d = half_digit(s.h[h], i);
            if (!d) continue;
            Pt q = tab[(d < 0 ? -d : d) - 1];
            if (h) q = Endo<C>::apply(q);
            if ((d < 0) != s.neg[h]) q = C::neg(q);
            C::add(acc, q);
        }
    }
    return acc;
}

// pts[i] = k_i pts[i] in place (affine), k_i = scalars[i], times c (Montgomery) when c is given; one point per thread
template <class C, class F>
__global__ void __launch_bounds__(128) points_scale_kernel(void* __restrict__ pts, uint32_t n, const fe* __restrict__ scalars,
                                                           const fe* __restrict__ c) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe k = fe_load(&scalars[i]);
    if (c) k = Fr::mul(k, *c);                          // canonical x Montgomery = the canonical product
    const typename C::Aff p = aff_load<F>(pts, i);
    typename C::Aff r;
    if (C::aff_is_inf(p) || fe_is_zero(k)) { r.x = F::zero(); r.y = F::zero(); }
    else r = C::to_affine(scale_point<C>(p, k.l));
    aff_store<F>(pts, i, r);
}

// test op 54: per scalar the G1 split then the G2 split, each half as 32 B two's complement
__global__ void __launch_bounds__(64) scale_split_kernel(const fe* __restrict__ k, uint32_t n, uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fe x = fe_load(&k[i]);
    const Split s[2] = {glv_split(x.l), gls_split(x.l)};
    for (int g = 0; g < 2; g++)
        for (int h = 0; h < 2; h++) {
            uint32_t w[8] = {s[g].h[h][0], s[g].h[h][1], s[g].h[h][2], s[g].h[h][3], 0, 0, 0, 0};
            if (s[g].neg[h]) mp_neg<8>(w);
            for (int j = 0; j < 8; j++) out[(size_t)i * 32 + 16 * g + 8 * h + j] = w[j];
        }
}

void scale_split_test_op(cudaStream_t st, const void* a, size_t n, void* out) {
    if (!a || !out) throw_error(B2G_E_SHAPE, "bad arguments");
    if (n == 0) return;
    struct Bufs { uint8_t *a = nullptr, *o = nullptr; ~Bufs() { if (a) cudaFree(a); if (o) cudaFree(o); } } d;
    d.a = dev_upload<uint8_t>(a, n * 32, st);
    CUDA_CHECK(cudaMalloc(&d.o, n * 128));
    scale_split_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>((const fe*)d.a, (uint32_t)n, (uint32_t*)d.o);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d.o, n * 128, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ---------------------------------------------------------------------------------------------- host side
// where the scalars of a pass come from: host (n x 32 B canonical), or the device powers c t^(i) of t (Montgomery)
struct ScaleScalars {
    const uint8_t* host = nullptr;
    const fe* t = nullptr;
    const fe* c = nullptr;                              // Montgomery multiplier, or none
    fe* d_k = nullptr;                                  // one slice of scalars (device)
    fe* d_pw = nullptr;                                 // the powers kernels' two words (device)
};

// one streamed pass: out[i] = k_i in[i] over count host points; with bad, the point rules of b2g_powers_check on every slice
static void scale_pass(Staging& sg, bool g2, const void* in, void* out, uint64_t count, const ScaleScalars& sc, bool gen,
                       unsigned long long* bad) {
    const size_t row = g2 ? 128 : 64;
    cudaStream_t st = sg.st;
    uint64_t prev_off = 0;
    uint32_t prev_cnt = 0;
    auto drain = [&](int b) {                           // the previous slice's points, from its pinned buffer to `out`
        CUDA_CHECK(cudaEventSynchronize(sg.used[b]));
        memcpy((uint8_t*)out + prev_off * row, sg.host[b], (size_t)prev_cnt * row);
    };
    uint64_t k = 0;
    for (uint64_t off = 0; off < count; off += POWERS_SLICE, k++) {
        const uint32_t cnt = (uint32_t)std::min<uint64_t>(POWERS_SLICE, count - off);
        const int b = (int)(k & 1);
        uint8_t* d = sg.upload(b, (const uint8_t*)in + off * row, (size_t)cnt * row);
        if (bad) powers_rules(g2, d, cnt, off, gen, bad, st);
        if (sc.host) CUDA_CHECK(cudaMemcpyAsync(sc.d_k, sc.host + off * 32, (size_t)cnt * 32, cudaMemcpyHostToDevice, st));
        else powers_scalars(sc.t, off, cnt, sc.d_pw, sc.d_k, st);
        const unsigned blocks = (cnt + 127) / 128;
        if (g2) points_scale_kernel<G2, Fq2><<<blocks, 128, 0, st>>>(d, cnt, sc.d_k, sc.c);
        else points_scale_kernel<G1, Fq><<<blocks, 128, 0, st>>>(d, cnt, sc.d_k, sc.c);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(sg.host[b], d, (size_t)cnt * row, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaEventRecord(sg.used[b], st));
        if (k) drain(b ^ 1);
        prev_off = off;
        prev_cnt = cnt;
    }
    if (k) drain((int)((k - 1) & 1));
}

static void points_scale_run(b2g_ctx* ctx, int g2, size_t n, const void* pts, const void* scalars, void* out) {
    if (!ctx || (n && (!pts || !scalars || !out))) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    const uint8_t* s = (const uint8_t*)scalars;
    for (size_t i = 0; i < n; i++)                      // k_i < r: the split's bounds need it
        if (!below(s + 32 * i, R_WORDS)) throw_error(B2G_E_INPUT, "scalars[" + std::to_string(i) + "] is not below r");
    if (n == 0) return;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    const size_t cap = std::min<size_t>(n, POWERS_SLICE);
    DevArena mem(st, true);
    ScaleScalars sc;
    sc.d_k = mem.alloc<fe>(cap * sizeof(fe));
    Staging sg(cap * (g2 ? 128 : 64), st);
    sc.host = s;
    scale_pass(sg, g2 != 0, pts, out, n, sc, false, nullptr);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

static void powers_contribute_run(b2g_ctx* ctx, const b2g_powers_desc* pw, const b2g_powers_secrets* sec, const b2g_powers_out* o) {
    if (!ctx || !pw || !sec || !o) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    const uint32_t p = pw->log_size;
    if (p < 1 || p > 28) throw_error(B2G_E_DOMAIN, "b2g_powers_contribute: log_size " + std::to_string(p) + " is outside 1..28");
    powers_arrays(pw, true);
    if (!o->tau_g1 || !o->tau_g2 || !o->alpha_tau_g1 || !o->beta_tau_g1 || !o->beta_g2) throw_error(B2G_E_SHAPE, "null output array");
    if (!sec->tau || !sec->alpha || !sec->beta) throw_error(B2G_E_SHAPE, "null secret");
    const uint64_t n = 1ull << p;
    struct Array { const char* name; const void* in; void* out; uint64_t count; bool g2, gen; int c; };
    const Array arrays[5] = {{"tau_g1", pw->tau_g1, o->tau_g1, 2 * n - 1, false, true, -1},
                             {"tau_g2", pw->tau_g2, o->tau_g2, n, true, true, -1},
                             {"alpha_tau_g1", pw->alpha_tau_g1, o->alpha_tau_g1, n, false, false, 1},
                             {"beta_tau_g1", pw->beta_tau_g1, o->beta_tau_g1, n, false, false, 2},
                             {"beta_g2", pw->beta_g2, o->beta_g2, 1, true, false, 2}};
    for (const Array& x : arrays)
        for (const Array& y : arrays)
            if (overlaps(x.out, x.count * (x.g2 ? 128 : 64), y.in, y.count * (y.g2 ? 128 : 64)))
                throw_error(B2G_E_SHAPE, std::string("b2g_powers_contribute: the output ") + x.name + " overlaps the input " + y.name);
    static const char* const NAMES[3] = {"tau", "alpha", "beta"};
    const void* secs[3] = {sec->tau, sec->alpha, sec->beta};
    for (int j = 0; j < 3; j++)
        if (!scalar_ok((const uint8_t*)secs[j])) throw_error(B2G_E_INPUT, std::string("secret ") + NAMES[j] + " is 0 or >= r");

    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    const uint64_t most = std::min<uint64_t>(2 * n - 1, POWERS_SLICE);
    // the secrets (canonical, then Montgomery), the powers kernels' words, and one slice of per-point scalars
    DevArena mem(st, true);
    fe* d_canon = mem.alloc<fe>(6 * sizeof(fe) + 2 * sizeof(fe));
    fe* d_mont = d_canon + 3;
    fe* d_scal = mem.alloc<fe>((most + 16) * sizeof(fe));
    upload_secrets(d_canon, secs, 3, st);
    to_mont(d_canon, 3, d_mont, st);
    CUDA_CHECK(cudaMemsetAsync(d_canon, 0, 3 * sizeof(fe), st));   // only the Montgomery forms are read from here on

    uint8_t* small = mem.alloc(128 + 64 + 8 * 5);     // the failing point, its rule, the lowest failing index per array
    unsigned long long* d_bad = (unsigned long long*)(small + 192);
    CUDA_CHECK(cudaMemsetAsync(d_bad, 0xff, 8 * 5, st));
    Staging sg(std::max<size_t>(most * 64, std::min<uint64_t>(n, POWERS_SLICE) * 128), st);
    ScaleScalars sc;
    sc.t = d_mont;
    sc.d_k = d_scal;
    sc.d_pw = d_mont + 3;
    for (int a = 0; a < 5; a++) {
        const Array& x = arrays[a];
        sc.c = x.c < 0 ? nullptr : d_mont + x.c;
        scale_pass(sg, x.g2, x.in, x.out, x.count, sc, x.gen, d_bad + a);
        uint64_t bad = 0;
        CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad + a, 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (bad >= x.count) continue;
        const uint32_t rule = bad_point_rule("b2g_powers_contribute", x.in, bad, x.g2, x.gen, small, (uint32_t*)(small + 128), st);
        static const char* const RULES[6] = {"", "a coordinate >= p", "off the curve", "at infinity", "not in G2", "not the generator"};
        throw_error(B2G_E_INPUT, std::string(x.name) + "[" + std::to_string(bad) + "]: " + (rule == 2 && x.g2 ? "off the twist" : RULES[rule]));
    }
    CUDA_CHECK(cudaStreamSynchronize(st));
}

}  // namespace b2g

extern "C" {

int b2g_points_scale(b2g_ctx* ctx, int g2, size_t n, const void* points, const void* scalars_canon, void* out) {
    return b2g::guarded_clear([&] { b2g::points_scale_run(ctx, g2, n, points, scalars_canon, out); });
}

int b2g_powers_contribute(b2g_ctx* ctx, const b2g_powers_desc* in, const b2g_powers_secrets* secrets, const b2g_powers_out* out) {
    return b2g::guarded_clear([&] { b2g::powers_contribute_run(ctx, in, secrets, out); });
}

}  // extern "C"
