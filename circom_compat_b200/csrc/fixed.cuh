// fixed.cuh - fixed-base scalar multiplication from 8-bit window tables, shared by the proof glue (prover.cu) and the
// verifier's prepared inputs (verify.cu): the table of a point P holds d * 256^w * P for every window w < 32 and digit
// d = 1..255 (32 x 255 affine points), and k * P is 32 look-ups and a 5-level tree inside one warp.
#pragma once
#include "ec.cuh"

namespace b2g {

// k * P from the 8-bit window table of P: lane w looks up digit w, a shared-memory tree adds the 32 partial points
template <class C, class F>
__device__ __forceinline__ typename C::Pt warp_fixed_mul(const void* __restrict__ table, const uint32_t* k, typename C::Pt* sh) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t byte = (k[lane >> 2] >> (8 * (lane & 3))) & 255u;
    typename C::Pt v = C::infinity();
    if (byte) v = C::from_affine(aff_load<F>(table, (size_t)lane * 255u + byte - 1u));
    sh[lane] = v;
    __syncwarp();
    #pragma unroll 1
    for (int d = 16; d > 0; d >>= 1) {
        if ((int)lane < d) { typename C::Pt a = sh[lane]; typename C::Pt q = sh[lane + d]; C::add(a, q); sh[lane] = a; }
        __syncwarp();
    }
    return sh[0];
}

__device__ __forceinline__ fe fe_from_words(uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t a4, uint32_t a5, uint32_t a6, uint32_t a7) {
    fe r; r.l[0] = a0; r.l[1] = a1; r.l[2] = a2; r.l[3] = a3; r.l[4] = a4; r.l[5] = a5; r.l[6] = a6; r.l[7] = a7; return r;
}
// standard generators: G1 = (1, 2); G2 = /root/reference/src/zkey.rs:443-463
__device__ __forceinline__ G1::Aff g1_generator() { G1::Aff g; g.x = Fq::one(); g.y = Fq::add(g.x, g.x); return g; }
__device__ __forceinline__ G2::Aff g2_generator() {
    G2::Aff g;
    g.x.c0 = Fq::from_canonical(fe_from_words(0xd992f6edu, 0x46debd5cu, 0xf75edaddu, 0x674322d4u, 0x5e5c4479u, 0x426a0066u, 0x121f1e76u, 0x1800deefu));
    g.x.c1 = Fq::from_canonical(fe_from_words(0xaef312c2u, 0x97e485b7u, 0x35a9e712u, 0xf1aa4933u, 0x31fb5d25u, 0x7260bfb7u, 0x920d483au, 0x198e9393u));
    g.y.c0 = Fq::from_canonical(fe_from_words(0x66fa7daau, 0x4ce6cc01u, 0x0c43d37bu, 0xe3d1e769u, 0x8dcb408fu, 0x4aab7180u, 0xdb8c6debu, 0x12c85ea5u));
    g.y.c1 = Fq::from_canonical(fe_from_words(0xd122975bu, 0x55acdadcu, 0x70b38ef3u, 0xbc4b3133u, 0x690c3395u, 0xec9e99adu, 0x585ff075u, 0x090689d0u));
    return g;
}
template <class C> struct Gen;
template <> struct Gen<G1> { static __device__ __forceinline__ G1::Aff get() { return g1_generator(); } };
template <> struct Gen<G2> { static __device__ __forceinline__ G2::Aff get() { return g2_generator(); } };

// entry i < 32 x 255 of a window table: table[w][d-1] = d * 256^w * G (affine), w = i / 255, d = i % 255 + 1
// base = nullptr: the group generator; else the affine point at `base` (e.g. delta of a proving key)
template <class C, class F>
__device__ __forceinline__ void fixed_table_entry(void* __restrict__ table, const void* __restrict__ base, uint32_t i) {
    uint32_t w = i / 255u, d = i % 255u + 1u;
    uint32_t k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    k[w >> 2] = d << (8 * (w & 3));
    typename C::Aff g = base ? aff_load<F>(base, 0) : Gen<C>::get();
    typename C::Pt p = C::mul_scalar(C::from_affine(g), k);
    aff_store<F>(table, i, C::to_affine(p));
}

// the whole window table of G, one entry per thread
template <class C, class F>
__global__ void fixed_table_kernel(void* __restrict__ table, const void* __restrict__ base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 32u * 255u) return;
    fixed_table_entry<C, F>(table, base, i);
}

// out[i] = scalars[i] * G (affine) for the window table of G and canonical scalars, one product per thread
template <class C, class F>
__global__ void __launch_bounds__(128) fixed_base_kernel(const void* __restrict__ table, const fe* __restrict__ scalars, uint32_t n, void* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe k = fe_load_nc(&scalars[i]);
    typename C::Pt acc = C::infinity();
    for (int w = 0; w < 32; w++) {
        uint32_t byte = (k.l[w >> 2] >> (8 * (w & 3))) & 255u;
        if (byte) C::madd(acc, aff_load<F>(table, (size_t)w * 255u + byte - 1u));
    }
    aff_store<F>(out, i, C::to_affine(acc));
}

}  // namespace b2g
