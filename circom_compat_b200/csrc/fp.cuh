// fp.cuh - 254-bit prime-field arithmetic for BN254 (Fq base field, Fr scalar field) on sm_90a.
//
// Replaces, on the device, what ark-ff 0.5.0's Fp256<MontBackend> (+asm, /root/reference/Cargo.toml:25) does on the
// CPU for the prover hot path.  Representation: 8 x 32-bit limbs, little-endian, Montgomery form with R = 2^256 -
// bit-identical in memory to the 4 x u64 LE Montgomery words the zkey stores (/root/reference/src/zkey.rs:327-332),
// so proving-key sections are uploaded without any conversion.
//
// The Montgomery product is a CIOS loop on two half-width accumulators ("even"/"odd" columns) so that every
// 32x32->64 partial product is one mad.lo.cc/madc.hi.cc pair (one IMAD.WIDE after ptxas) and every carry chain lives
// inside a single asm block.  All results are fully reduced to [0, p).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b2g {

struct alignas(32) fe { uint32_t l[8]; };

// ---------------------------------------------------------------------------------------------- moduli
struct FqParams {
    // q = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
    static constexpr uint32_t P0 = 0xd87cfd47u, P1 = 0x3c208c16u, P2 = 0x6871ca8du, P3 = 0x97816a91u,
                              P4 = 0x8181585du, P5 = 0xb85045b6u, P6 = 0xe131a029u, P7 = 0x30644e72u;
    static constexpr uint32_t INV = 0xe4866389u;              // -q^-1 mod 2^32
    // R mod q (Montgomery one)
    static constexpr uint32_t R0 = 0xc58f0d9du, R1 = 0xd35d438du, R2 = 0xf5c70b3du, R3 = 0x0a78eb28u,
                              R4 = 0x7879462cu, R5 = 0x666ea36fu, R6 = 0x9a07df2fu, R7 = 0x0e0a77c1u;
    // R^2 mod q
    static constexpr uint32_t RR0 = 0x538afa89u, RR1 = 0xf32cfc5bu, RR2 = 0xd44501fbu, RR3 = 0xb5e71911u,
                              RR4 = 0x0a417ff6u, RR5 = 0x47ab1effu, RR6 = 0xcab8351fu, RR7 = 0x06d89f71u;
};
struct FrParams {
    // r = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
    static constexpr uint32_t P0 = 0xf0000001u, P1 = 0x43e1f593u, P2 = 0x79b97091u, P3 = 0x2833e848u,
                              P4 = 0x8181585du, P5 = 0xb85045b6u, P6 = 0xe131a029u, P7 = 0x30644e72u;
    static constexpr uint32_t INV = 0xefffffffu;
    static constexpr uint32_t R0 = 0x4ffffffbu, R1 = 0xac96341cu, R2 = 0x9f60cd29u, R3 = 0x36fc7695u,
                              R4 = 0x7879462eu, R5 = 0x666ea36fu, R6 = 0x9a07df2fu, R7 = 0x0e0a77c1u;
    static constexpr uint32_t RR0 = 0xae216da7u, RR1 = 0x1bb8e645u, RR2 = 0xe35c59e3u, RR3 = 0x53fe3ab1u,
                              RR4 = 0x53bb8085u, RR5 = 0x8c49833du, RR6 = 0x7f4e44a5u, RR7 = 0x0216d0b1u;
};

// ---------------------------------------------------------------------------------------------- raw helpers
__device__ __forceinline__ bool fe_is_zero(const fe& a) {
    return (a.l[0] | a.l[1] | a.l[2] | a.l[3] | a.l[4] | a.l[5] | a.l[6] | a.l[7]) == 0u;
}
__device__ __forceinline__ bool fe_equal(const fe& a, const fe& b) {
    return ((a.l[0] ^ b.l[0]) | (a.l[1] ^ b.l[1]) | (a.l[2] ^ b.l[2]) | (a.l[3] ^ b.l[3]) |
            (a.l[4] ^ b.l[4]) | (a.l[5] ^ b.l[5]) | (a.l[6] ^ b.l[6]) | (a.l[7] ^ b.l[7])) == 0u;
}
__device__ __forceinline__ fe fe_zero() {
    fe r;
    r.l[0] = 0; r.l[1] = 0; r.l[2] = 0; r.l[3] = 0; r.l[4] = 0; r.l[5] = 0; r.l[6] = 0; r.l[7] = 0;
    return r;
}

// 256-bit loads/stores of one element (32-byte aligned)
__device__ __forceinline__ fe fe_load(const void* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    fe r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
// read-only (non-coherent) load of one element: two 128-bit LDG.CONSTANT (sm_90 has no 256-bit global load).
__device__ __forceinline__ fe fe_load_nc(const void* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    fe r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
__device__ __forceinline__ void fe_store(void* p, const fe& v) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// ---------------------------------------------------------------------------------------------- the field
template <class P>
struct Fp {
    using elem = fe;

    static __device__ __forceinline__ fe zero() { return fe_zero(); }
    static __device__ __forceinline__ fe one() {
        fe r; r.l[0] = P::R0; r.l[1] = P::R1; r.l[2] = P::R2; r.l[3] = P::R3; r.l[4] = P::R4; r.l[5] = P::R5; r.l[6] = P::R6; r.l[7] = P::R7;
        return r;
    }
    static __device__ __forceinline__ fe r2() {
        fe r; r.l[0] = P::RR0; r.l[1] = P::RR1; r.l[2] = P::RR2; r.l[3] = P::RR3; r.l[4] = P::RR4; r.l[5] = P::RR5; r.l[6] = P::RR6; r.l[7] = P::RR7;
        return r;
    }
    static __device__ __forceinline__ bool is_zero(const fe& a) { return fe_is_zero(a); }
    static __device__ __forceinline__ bool eq(const fe& a, const fe& b) { return fe_equal(a, b); }

    // r = a - p if a >= p else a     (a < 2p)
    static __device__ __forceinline__ fe reduce_once(const fe& a) {
        fe t; uint32_t br;
        asm("sub.cc.u32 %0, %9, %17;\n\t"
            "subc.cc.u32 %1, %10, %18;\n\t"
            "subc.cc.u32 %2, %11, %19;\n\t"
            "subc.cc.u32 %3, %12, %20;\n\t"
            "subc.cc.u32 %4, %13, %21;\n\t"
            "subc.cc.u32 %5, %14, %22;\n\t"
            "subc.cc.u32 %6, %15, %23;\n\t"
            "subc.cc.u32 %7, %16, %24;\n\t"
            "subc.u32 %8, 0, 0;"
            : "=r"(t.l[0]), "=r"(t.l[1]), "=r"(t.l[2]), "=r"(t.l[3]), "=r"(t.l[4]), "=r"(t.l[5]), "=r"(t.l[6]), "=r"(t.l[7]), "=r"(br)
            : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
              "n"(P::P0), "n"(P::P1), "n"(P::P2), "n"(P::P3), "n"(P::P4), "n"(P::P5), "n"(P::P6), "n"(P::P7));
        fe r;
        #pragma unroll
        for (int i = 0; i < 8; i++) r.l[i] = br ? a.l[i] : t.l[i];
        return r;
    }

    static __device__ __forceinline__ fe add(const fe& a, const fe& b) {
        fe s;
        asm("add.cc.u32 %0, %8, %16;\n\t"
            "addc.cc.u32 %1, %9, %17;\n\t"
            "addc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\t"
            "addc.cc.u32 %4, %12, %20;\n\t"
            "addc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\t"
            "addc.u32 %7, %15, %23;"
            : "=r"(s.l[0]), "=r"(s.l[1]), "=r"(s.l[2]), "=r"(s.l[3]), "=r"(s.l[4]), "=r"(s.l[5]), "=r"(s.l[6]), "=r"(s.l[7])
            : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
              "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
        return reduce_once(s);      // a, b < p < 2^254  =>  no carry out of limb 7
    }
    static __device__ __forceinline__ fe dbl(const fe& a) { return add(a, a); }

    static __device__ __forceinline__ fe sub(const fe& a, const fe& b) {
        fe d; uint32_t br;
        asm("sub.cc.u32 %0, %9, %17;\n\t"
            "subc.cc.u32 %1, %10, %18;\n\t"
            "subc.cc.u32 %2, %11, %19;\n\t"
            "subc.cc.u32 %3, %12, %20;\n\t"
            "subc.cc.u32 %4, %13, %21;\n\t"
            "subc.cc.u32 %5, %14, %22;\n\t"
            "subc.cc.u32 %6, %15, %23;\n\t"
            "subc.cc.u32 %7, %16, %24;\n\t"
            "subc.u32 %8, 0, 0;"
            : "=r"(d.l[0]), "=r"(d.l[1]), "=r"(d.l[2]), "=r"(d.l[3]), "=r"(d.l[4]), "=r"(d.l[5]), "=r"(d.l[6]), "=r"(d.l[7]), "=r"(br)
            : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
              "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
        // br = 0xffffffff when a < b: add p back
        uint32_t m0 = P::P0 & br, m1 = P::P1 & br, m2 = P::P2 & br, m3 = P::P3 & br,
                 m4 = P::P4 & br, m5 = P::P5 & br, m6 = P::P6 & br, m7 = P::P7 & br;
        asm("add.cc.u32 %0, %0, %8;\n\t"
            "addc.cc.u32 %1, %1, %9;\n\t"
            "addc.cc.u32 %2, %2, %10;\n\t"
            "addc.cc.u32 %3, %3, %11;\n\t"
            "addc.cc.u32 %4, %4, %12;\n\t"
            "addc.cc.u32 %5, %5, %13;\n\t"
            "addc.cc.u32 %6, %6, %14;\n\t"
            "addc.u32 %7, %7, %15;"
            : "+r"(d.l[0]), "+r"(d.l[1]), "+r"(d.l[2]), "+r"(d.l[3]), "+r"(d.l[4]), "+r"(d.l[5]), "+r"(d.l[6]), "+r"(d.l[7])
            : "r"(m0), "r"(m1), "r"(m2), "r"(m3), "r"(m4), "r"(m5), "r"(m6), "r"(m7));
        return d;
    }
    static __device__ __forceinline__ fe neg(const fe& a) { return sub(zero(), a); }

    // ------------------------------------------------------------------ Montgomery product
    // acc[0..7] = { lo,hi of x0*b ; x1*b ; x2*b ; x3*b }
    static __device__ __forceinline__ void mul4(uint32_t* acc, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t b) {
        // mul.wide.u32 is ONE IMAD.WIDE; a mul.lo/mul.hi pair without a carry chain is left unfused by ptxas (IMAD + IMAD.HI)
        asm("{\n\t.reg .u64 t0, t1, t2, t3;\n\t"
            "mul.wide.u32 t0, %8, %12;\n\t mul.wide.u32 t1, %9, %12;\n\t"
            "mul.wide.u32 t2, %10, %12;\n\t mul.wide.u32 t3, %11, %12;\n\t"
            "mov.b64 {%0, %1}, t0;\n\t mov.b64 {%2, %3}, t1;\n\t mov.b64 {%4, %5}, t2;\n\t mov.b64 {%6, %7}, t3;\n\t}"
            : "=r"(acc[0]), "=r"(acc[1]), "=r"(acc[2]), "=r"(acc[3]), "=r"(acc[4]), "=r"(acc[5]), "=r"(acc[6]), "=r"(acc[7])
            : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(b));
    }
    // acc += { x0*b ; x1*b ; x2*b ; x3*b } as one 256-bit carry chain; the carry out is added to `top`
    static __device__ __forceinline__ void cmad4(uint32_t* acc, uint32_t& top, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t b) {
        asm("mad.lo.cc.u32 %0, %9, %13, %0;\n\t madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
            "madc.lo.cc.u32 %2, %10, %13, %2;\n\t madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
            "madc.lo.cc.u32 %4, %11, %13, %4;\n\t madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
            "madc.lo.cc.u32 %6, %12, %13, %6;\n\t madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
            "addc.u32 %8, %8, 0;"
            : "+r"(acc[0]), "+r"(acc[1]), "+r"(acc[2]), "+r"(acc[3]), "+r"(acc[4]), "+r"(acc[5]), "+r"(acc[6]), "+r"(acc[7]), "+r"(top)
            : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(b));
    }
    // same, carry out discarded (provably zero)
    static __device__ __forceinline__ void cmad4_nc(uint32_t* acc, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t b) {
        asm("mad.lo.cc.u32 %0, %8, %12, %0;\n\t madc.hi.cc.u32 %1, %8, %12, %1;\n\t"
            "madc.lo.cc.u32 %2, %9, %12, %2;\n\t madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
            "madc.lo.cc.u32 %4, %10, %12, %4;\n\t madc.hi.cc.u32 %5, %10, %12, %5;\n\t"
            "madc.lo.cc.u32 %6, %11, %12, %6;\n\t madc.hi.cc.u32 %7, %11, %12, %7;"
            : "+r"(acc[0]), "+r"(acc[1]), "+r"(acc[2]), "+r"(acc[3]), "+r"(acc[4]), "+r"(acc[5]), "+r"(acc[6]), "+r"(acc[7])
            : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(b));
    }
    // x0 += e[1] (carry into the chain);  e[j], e[j+1] = {x_odd * b} + e[j+2], e[j+3]  (in-place two-limb right shift)
    static __device__ __forceinline__ void madc_shift(uint32_t& x0, uint32_t* e, uint32_t a1, uint32_t a3, uint32_t a5, uint32_t a7, uint32_t b) {
        asm("add.cc.u32 %8, %8, %1;\n\t"
            "madc.lo.cc.u32 %0, %9, %13, %2;\n\t madc.hi.cc.u32 %1, %9, %13, %3;\n\t"
            "madc.lo.cc.u32 %2, %10, %13, %4;\n\t madc.hi.cc.u32 %3, %10, %13, %5;\n\t"
            "madc.lo.cc.u32 %4, %11, %13, %6;\n\t madc.hi.cc.u32 %5, %11, %13, %7;\n\t"
            "madc.lo.cc.u32 %6, %12, %13, 0;\n\t madc.hi.cc.u32 %7, %12, %13, 0;"
            : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0)
            : "r"(a1), "r"(a3), "r"(a5), "r"(a7), "r"(b));
    }

    // one CIOS row: x = array aligned to limb 0, e = array that becomes the limb-1-aligned one
    static __device__ __forceinline__ void row(uint32_t* x, uint32_t* e, const fe& a, uint32_t b, bool first) {
        if (first) {
            mul4(e, a.l[1], a.l[3], a.l[5], a.l[7], b);
            mul4(x, a.l[0], a.l[2], a.l[4], a.l[6], b);
        } else {
            madc_shift(x[0], e, a.l[1], a.l[3], a.l[5], a.l[7], b);
            cmad4(x, e[7], a.l[0], a.l[2], a.l[4], a.l[6], b);
        }
        uint32_t m = x[0] * P::INV;
        cmad4_nc(e, P::P1, P::P3, P::P5, P::P7, m);
        cmad4(x, e[7], P::P0, P::P2, P::P4, P::P6, m);
    }

    static __device__ __forceinline__ fe mul(const fe& a, const fe& b) {
        uint32_t ev[8], od[8];
        row(ev, od, a, b.l[0], true);
        row(od, ev, a, b.l[1], false);
        row(ev, od, a, b.l[2], false);
        row(od, ev, a, b.l[3], false);
        row(ev, od, a, b.l[4], false);
        row(od, ev, a, b.l[5], false);
        row(ev, od, a, b.l[6], false);
        row(od, ev, a, b.l[7], false);
        // after the last row: od is limb-0 aligned with od[0] == 0, ev is limb-1 aligned; result = ev + (od >> 32)
        fe r;
        asm("add.cc.u32 %0, %8, %16;\n\t"
            "addc.cc.u32 %1, %9, %17;\n\t"
            "addc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\t"
            "addc.cc.u32 %4, %12, %20;\n\t"
            "addc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\t"
            "addc.u32 %7, %15, 0;"
            : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
            : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
              "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
        return reduce_once(r);
    }
    // defined after the lazy-reduction blocks: sqr(a) = redc(sqr_wide(a)), 36 + 64 products instead of 128
    static __device__ __forceinline__ fe sqr(const fe& a) {
        uint32_t t[16];
        sqr_wide(t, a);
        return redc(t);
    }

    // ------------------------------------------------------------------ lazy-reduction building blocks (used by Fq2)
    // one row of the plain 256 x 32 product, same column bookkeeping as row() but without the reduction step:
    // after the call x[0] is a finished limb of the result and x[1..7], e[0..7] carry the rest one limb further up.
    static __device__ __forceinline__ void prow(uint32_t* x, uint32_t* e, const fe& a, uint32_t b, bool first) {
        if (first) {
            mul4(e, a.l[1], a.l[3], a.l[5], a.l[7], b);
            mul4(x, a.l[0], a.l[2], a.l[4], a.l[6], b);
        } else {
            madc_shift(x[0], e, a.l[1], a.l[3], a.l[5], a.l[7], b);
            cmad4(x, e[7], a.l[0], a.l[2], a.l[4], a.l[6], b);
        }
    }
    // t[0..15] = a * b as a plain 512-bit integer, a < 2^255 (so that the top column never overflows), b any 256-bit
    // value.  Eight rows; each retires one low limb, so there is one closing addc per row and no zero-initialisation.
    static __device__ __forceinline__ void mul_wide(uint32_t* t, const fe& a, const fe& b) {
        uint32_t ev[8], od[8];
        prow(ev, od, a, b.l[0], true);  t[0] = ev[0];
        prow(od, ev, a, b.l[1], false); t[1] = od[0];
        prow(ev, od, a, b.l[2], false); t[2] = ev[0];
        prow(od, ev, a, b.l[3], false); t[3] = od[0];
        prow(ev, od, a, b.l[4], false); t[4] = ev[0];
        prow(od, ev, a, b.l[5], false); t[5] = od[0];
        prow(ev, od, a, b.l[6], false); t[6] = ev[0];
        prow(od, ev, a, b.l[7], false); t[7] = od[0];
        // od is limb-7 aligned with od[0] retired, ev is limb-8 aligned: high half = ev + (od >> 32)
        asm("add.cc.u32 %0, %8, %16;\n\t"
            "addc.cc.u32 %1, %9, %17;\n\t"
            "addc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\t"
            "addc.cc.u32 %4, %12, %20;\n\t"
            "addc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\t"
            "addc.u32 %7, %15, 0;"
            : "=r"(t[8]), "=r"(t[9]), "=r"(t[10]), "=r"(t[11]), "=r"(t[12]), "=r"(t[13]), "=r"(t[14]), "=r"(t[15])
            : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
              "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
    }

    // ---- squaring: a^2 = sum_j a_j 2^(32j) [ (a_j + topbit(a_(j-1))) 2^(32j) + sum_(i<j) b_i 2^(32i) ],  b = limbs of 2a.
    // 36 products instead of 64, no doubling pass; each carry chain ends on two fresh limbs, so nothing has to be closed.
    // f = x * y + add
    static __device__ __forceinline__ void chain1(uint32_t* f, uint32_t x, uint32_t y, uint32_t add) {
        asm("mad.lo.cc.u32 %0, %2, %3, %4;\n\t madc.hi.u32 %1, %2, %3, 0;" : "=&r"(f[0]), "=&r"(f[1]) : "r"(x), "r"(y), "r"(add));
    }
    // acc[0..1] += x0 * y ; acc[2..3] = x1 * y + add (+ carry)
    static __device__ __forceinline__ void chain2(uint32_t* acc, uint32_t x0, uint32_t x1, uint32_t y, uint32_t add) {
        asm("mad.lo.cc.u32 %0, %4, %6, %0;\n\t madc.hi.cc.u32 %1, %4, %6, %1;\n\t"
            "madc.lo.cc.u32 %2, %5, %6, %7;\n\t madc.hi.u32 %3, %5, %6, 0;"
            : "+r"(acc[0]), "+r"(acc[1]), "=&r"(acc[2]), "=&r"(acc[3]) : "r"(x0), "r"(x1), "r"(y), "r"(add));
    }
    static __device__ __forceinline__ void chain3(uint32_t* acc, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t y, uint32_t add) {
        asm("mad.lo.cc.u32 %0, %6, %9, %0;\n\t madc.hi.cc.u32 %1, %6, %9, %1;\n\t"
            "madc.lo.cc.u32 %2, %7, %9, %2;\n\t madc.hi.cc.u32 %3, %7, %9, %3;\n\t"
            "madc.lo.cc.u32 %4, %8, %9, %10;\n\t madc.hi.u32 %5, %8, %9, 0;"
            : "+r"(acc[0]), "+r"(acc[1]), "+r"(acc[2]), "+r"(acc[3]), "=&r"(acc[4]), "=&r"(acc[5])
            : "r"(x0), "r"(x1), "r"(x2), "r"(y), "r"(add));
    }
    static __device__ __forceinline__ void chain4(uint32_t* acc, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t y, uint32_t add) {
        asm("mad.lo.cc.u32 %0, %8, %12, %0;\n\t madc.hi.cc.u32 %1, %8, %12, %1;\n\t"
            "madc.lo.cc.u32 %2, %9, %12, %2;\n\t madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
            "madc.lo.cc.u32 %4, %10, %12, %4;\n\t madc.hi.cc.u32 %5, %10, %12, %5;\n\t"
            "madc.lo.cc.u32 %6, %11, %12, %13;\n\t madc.hi.u32 %7, %11, %12, 0;"
            : "+r"(acc[0]), "+r"(acc[1]), "+r"(acc[2]), "+r"(acc[3]), "+r"(acc[4]), "+r"(acc[5]), "=&r"(acc[6]), "=&r"(acc[7])
            : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y), "r"(add));
    }
    // t[0..15] = a^2 (any 256-bit a)
    static __device__ __forceinline__ void sqr_wide(uint32_t* t, const fe& a) {
        uint32_t b[7], m[8], ev[16], od[14];
        b[0] = a.l[0] << 1;
        #pragma unroll
        for (int i = 1; i < 7; i++) b[i] = __funnelshift_l(a.l[i - 1], a.l[i], 1);
        #pragma unroll
        for (int j = 1; j < 8; j++) m[j] = a.l[j] & (uint32_t)((int32_t)a.l[j - 1] >> 31);
        // columns at even limb positions: a_j * (b_i, i = j-2, j-4, ...) then a_j * a_j + m_j on fresh limbs 2j, 2j+1
        chain1(&ev[0], a.l[0], a.l[0], 0);
        chain1(&ev[2], a.l[1], a.l[1], m[1]);
        chain2(&ev[2], b[0], a.l[2], a.l[2], m[2]);
        chain2(&ev[4], b[1], a.l[3], a.l[3], m[3]);
        chain3(&ev[4], b[0], b[2], a.l[4], a.l[4], m[4]);
        chain3(&ev[6], b[1], b[3], a.l[5], a.l[5], m[5]);
        chain4(&ev[6], b[0], b[2], b[4], a.l[6], a.l[6], m[6]);
        chain4(&ev[8], b[1], b[3], b[5], a.l[7], a.l[7], m[7]);
        // columns at odd limb positions (od[k] sits at limb k + 1): a_j * (b_i, i = j-1, j-3, ...)
        chain1(&od[0], b[0], a.l[1], 0);
        chain1(&od[2], b[1], a.l[2], 0);
        chain2(&od[2], b[0], b[2], a.l[3], 0);
        chain2(&od[4], b[1], b[3], a.l[4], 0);
        chain3(&od[4], b[0], b[2], b[4], a.l[5], 0);
        chain3(&od[6], b[1], b[3], b[5], a.l[6], 0);
        chain4(&od[6], b[0], b[2], b[4], b[6], a.l[7], 0);
        t[0] = ev[0];
        asm("add.cc.u32 %0, %15, %30;\n\t"
            "addc.cc.u32 %1, %16, %31;\n\t"
            "addc.cc.u32 %2, %17, %32;\n\t"
            "addc.cc.u32 %3, %18, %33;\n\t"
            "addc.cc.u32 %4, %19, %34;\n\t"
            "addc.cc.u32 %5, %20, %35;\n\t"
            "addc.cc.u32 %6, %21, %36;\n\t"
            "addc.cc.u32 %7, %22, %37;\n\t"
            "addc.cc.u32 %8, %23, %38;\n\t"
            "addc.cc.u32 %9, %24, %39;\n\t"
            "addc.cc.u32 %10, %25, %40;\n\t"
            "addc.cc.u32 %11, %26, %41;\n\t"
            "addc.cc.u32 %12, %27, %42;\n\t"
            "addc.cc.u32 %13, %28, %43;\n\t"
            "addc.u32 %14, %29, 0;"
            : "=r"(t[1]), "=r"(t[2]), "=r"(t[3]), "=r"(t[4]), "=r"(t[5]), "=r"(t[6]), "=r"(t[7]), "=r"(t[8]),
              "=r"(t[9]), "=r"(t[10]), "=r"(t[11]), "=r"(t[12]), "=r"(t[13]), "=r"(t[14]), "=r"(t[15])
            : "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]), "r"(ev[8]),
              "r"(ev[9]), "r"(ev[10]), "r"(ev[11]), "r"(ev[12]), "r"(ev[13]), "r"(ev[14]), "r"(ev[15]),
              "r"(od[0]), "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]),
              "r"(od[8]), "r"(od[9]), "r"(od[10]), "r"(od[11]), "r"(od[12]), "r"(od[13]));
    }

    // t -= u  (512-bit); returns the borrow mask (0xffffffff when t < u)
    static __device__ __forceinline__ uint32_t sub_wide(uint32_t* t, const uint32_t* u) {
        uint32_t br;
        asm("sub.cc.u32 %0, %0, %17;\n\t"
            "subc.cc.u32 %1, %1, %18;\n\t"
            "subc.cc.u32 %2, %2, %19;\n\t"
            "subc.cc.u32 %3, %3, %20;\n\t"
            "subc.cc.u32 %4, %4, %21;\n\t"
            "subc.cc.u32 %5, %5, %22;\n\t"
            "subc.cc.u32 %6, %6, %23;\n\t"
            "subc.cc.u32 %7, %7, %24;\n\t"
            "subc.cc.u32 %8, %8, %25;\n\t"
            "subc.cc.u32 %9, %9, %26;\n\t"
            "subc.cc.u32 %10, %10, %27;\n\t"
            "subc.cc.u32 %11, %11, %28;\n\t"
            "subc.cc.u32 %12, %12, %29;\n\t"
            "subc.cc.u32 %13, %13, %30;\n\t"
            "subc.cc.u32 %14, %14, %31;\n\t"
            "subc.cc.u32 %15, %15, %32;\n\t"
            "subc.u32 %16, 0, 0;"
            : "+r"(t[0]), "+r"(t[1]), "+r"(t[2]), "+r"(t[3]), "+r"(t[4]), "+r"(t[5]), "+r"(t[6]), "+r"(t[7]),
              "+r"(t[8]), "+r"(t[9]), "+r"(t[10]), "+r"(t[11]), "+r"(t[12]), "+r"(t[13]), "+r"(t[14]), "+r"(t[15]), "=r"(br)
            : "r"(u[0]), "r"(u[1]), "r"(u[2]), "r"(u[3]), "r"(u[4]), "r"(u[5]), "r"(u[6]), "r"(u[7]),
              "r"(u[8]), "r"(u[9]), "r"(u[10]), "r"(u[11]), "r"(u[12]), "r"(u[13]), "r"(u[14]), "r"(u[15]));
        return br;
    }

    // high half of t += p & mask  (adds p * 2^256 when mask is all ones)
    static __device__ __forceinline__ void add_p_high(uint32_t* t, uint32_t mask) {
        uint32_t m0 = P::P0 & mask, m1 = P::P1 & mask, m2 = P::P2 & mask, m3 = P::P3 & mask,
                 m4 = P::P4 & mask, m5 = P::P5 & mask, m6 = P::P6 & mask, m7 = P::P7 & mask;
        asm("add.cc.u32 %0, %0, %8;\n\t"
            "addc.cc.u32 %1, %1, %9;\n\t"
            "addc.cc.u32 %2, %2, %10;\n\t"
            "addc.cc.u32 %3, %3, %11;\n\t"
            "addc.cc.u32 %4, %4, %12;\n\t"
            "addc.cc.u32 %5, %5, %13;\n\t"
            "addc.cc.u32 %6, %6, %14;\n\t"
            "addc.u32 %7, %7, %15;"
            : "+r"(t[8]), "+r"(t[9]), "+r"(t[10]), "+r"(t[11]), "+r"(t[12]), "+r"(t[13]), "+r"(t[14]), "+r"(t[15])
            : "r"(m0), "r"(m1), "r"(m2), "r"(m3), "r"(m4), "r"(m5), "r"(m6), "r"(m7));
    }

    // x0 += e[1]; m = x0 * INV; e[j], e[j+1] = {p_odd * m} + e[j+2], e[j+3]  (the reduction row's counterpart of madc_shift;
    // m is computed between the first add and the multiply-add chain, which mul.lo leaves the carry flag alone for)
    static __device__ __forceinline__ void madc_shift_m(uint32_t& x0, uint32_t* e, uint32_t& m) {
        asm("add.cc.u32 %8, %8, %1;\n\t"
            "mul.lo.u32 %9, %8, %10;\n\t"
            "madc.lo.cc.u32 %0, %11, %9, %2;\n\t madc.hi.cc.u32 %1, %11, %9, %3;\n\t"
            "madc.lo.cc.u32 %2, %12, %9, %4;\n\t madc.hi.cc.u32 %3, %12, %9, %5;\n\t"
            "madc.lo.cc.u32 %4, %13, %9, %6;\n\t madc.hi.cc.u32 %5, %13, %9, %7;\n\t"
            "madc.lo.cc.u32 %6, %14, %9, 0;\n\t madc.hi.u32 %7, %14, %9, 0;"
            : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0), "=&r"(m)
            : "r"(P::INV), "r"(P::P1), "r"(P::P3), "r"(P::P5), "r"(P::P7));
    }
    // one reduction row: x is limb-0 aligned, e becomes the limb-1 aligned array; x[0] ends up 0
    static __device__ __forceinline__ void mrow(uint32_t* x, uint32_t* e) {
        uint32_t m;
        madc_shift_m(x[0], e, m);
        cmad4(x, e[7], P::P0, P::P2, P::P4, P::P6, m);
    }
    // Montgomery reduction of a 512-bit t < p * 2^256: returns (t + M p) / 2^256 reduced once, i.e. in [0, p)
    // (the value before the subtraction is < t / 2^256 + p < 2p).  The low half is folded with the same even/odd column
    // rows as mul(); the high half is added at the end.
    static __device__ __forceinline__ fe redc(const uint32_t* t) {
        uint32_t ev[8], od[8];
        #pragma unroll
        for (int i = 0; i < 8; i++) ev[i] = t[i];
        {
            const uint32_t m = ev[0] * P::INV;
            mul4(od, P::P1, P::P3, P::P5, P::P7, m);
            cmad4(ev, od[7], P::P0, P::P2, P::P4, P::P6, m);
        }
        mrow(od, ev); mrow(ev, od); mrow(od, ev); mrow(ev, od); mrow(od, ev); mrow(ev, od); mrow(od, ev);
        // od is limb-0 aligned with od[0] == 0, ev is limb-1 aligned: r = ev + (od >> 32) + t[8..15]   (< 2p, no carry out)
        fe r;
        asm("add.cc.u32 %0, %8, %16;\n\t"
            "addc.cc.u32 %1, %9, %17;\n\t"
            "addc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\t"
            "addc.cc.u32 %4, %12, %20;\n\t"
            "addc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\t"
            "addc.u32 %7, %15, 0;"
            : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
            : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
              "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
        asm("add.cc.u32 %0, %0, %8;\n\t"
            "addc.cc.u32 %1, %1, %9;\n\t"
            "addc.cc.u32 %2, %2, %10;\n\t"
            "addc.cc.u32 %3, %3, %11;\n\t"
            "addc.cc.u32 %4, %4, %12;\n\t"
            "addc.cc.u32 %5, %5, %13;\n\t"
            "addc.cc.u32 %6, %6, %14;\n\t"
            "addc.u32 %7, %7, %15;"
            : "+r"(r.l[0]), "+r"(r.l[1]), "+r"(r.l[2]), "+r"(r.l[3]), "+r"(r.l[4]), "+r"(r.l[5]), "+r"(r.l[6]), "+r"(r.l[7])
            : "r"(t[8]), "r"(t[9]), "r"(t[10]), "r"(t[11]), "r"(t[12]), "r"(t[13]), "r"(t[14]), "r"(t[15]));
        return reduce_once(r);
    }

    // Column form of the same product: sixteen independent 8-limb chains on zero-initialised even/odd accumulators.  More
    // ALU instructions and live registers than mul_wide() but no row-to-row dependency; the called Fq2::mul uses it for the
    // latency-bound single-thread chains (fold, reduce, glue).
    static __device__ __forceinline__ void mul_wide_cols(uint32_t* t, const fe& a, const fe& b) {
        uint32_t ev[17], od[16];
        #pragma unroll
        for (int i = 0; i < 17; i++) ev[i] = 0;
        #pragma unroll
        for (int i = 0; i < 16; i++) od[i] = 0;
        #pragma unroll
        for (int i = 0; i < 8; i += 2) {
            // even row i: a_even * b_i -> positions i.. (ev), a_odd * b_i -> positions i+1.. (od index i)
            cmad4(&ev[i], ev[i + 8], a.l[0], a.l[2], a.l[4], a.l[6], b.l[i]);
            cmad4(&od[i], od[i + 8 < 16 ? i + 8 : 15], a.l[1], a.l[3], a.l[5], a.l[7], b.l[i]);
            // odd row i+1: a_even * b -> positions i+1.. (od index i), a_odd * b -> positions i+2.. (ev)
            cmad4(&od[i], od[i + 8 < 16 ? i + 8 : 15], a.l[0], a.l[2], a.l[4], a.l[6], b.l[i + 1]);
            cmad4(&ev[i + 2], ev[i + 10 < 17 ? i + 10 : 16], a.l[1], a.l[3], a.l[5], a.l[7], b.l[i + 1]);
        }
        // t = ev + (od << 32)
        t[0] = ev[0];
        asm("add.cc.u32 %0, %15, %30;\n\t"
            "addc.cc.u32 %1, %16, %31;\n\t"
            "addc.cc.u32 %2, %17, %32;\n\t"
            "addc.cc.u32 %3, %18, %33;\n\t"
            "addc.cc.u32 %4, %19, %34;\n\t"
            "addc.cc.u32 %5, %20, %35;\n\t"
            "addc.cc.u32 %6, %21, %36;\n\t"
            "addc.cc.u32 %7, %22, %37;\n\t"
            "addc.cc.u32 %8, %23, %38;\n\t"
            "addc.cc.u32 %9, %24, %39;\n\t"
            "addc.cc.u32 %10, %25, %40;\n\t"
            "addc.cc.u32 %11, %26, %41;\n\t"
            "addc.cc.u32 %12, %27, %42;\n\t"
            "addc.cc.u32 %13, %28, %43;\n\t"
            "addc.u32 %14, %29, %44;"
            : "=r"(t[1]), "=r"(t[2]), "=r"(t[3]), "=r"(t[4]), "=r"(t[5]), "=r"(t[6]), "=r"(t[7]), "=r"(t[8]),
              "=r"(t[9]), "=r"(t[10]), "=r"(t[11]), "=r"(t[12]), "=r"(t[13]), "=r"(t[14]), "=r"(t[15])
            : "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]), "r"(ev[8]),
              "r"(ev[9]), "r"(ev[10]), "r"(ev[11]), "r"(ev[12]), "r"(ev[13]), "r"(ev[14]), "r"(ev[15]),
              "r"(od[0]), "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]),
              "r"(od[8]), "r"(od[9]), "r"(od[10]), "r"(od[11]), "r"(od[12]), "r"(od[13]), "r"(od[14]));
    }

    // a*b - c*d with ONE Montgomery reduction (two 512-bit products, wide subtraction, + p*2^256 when negative)
    static __device__ __forceinline__ fe mul_sub(const fe& a, const fe& b, const fe& c, const fe& d) {
        uint32_t u[16], v[16];
        mul_wide(u, a, b);
        mul_wide(v, c, d);
        const uint32_t br = sub_wide(u, v);
        add_p_high(u, br);
        return redc(u);
    }

    static __device__ __forceinline__ fe from_canonical(const fe& a) { return mul(a, r2()); }
    static __device__ __forceinline__ fe to_canonical(const fe& a) {
        fe o = fe_zero(); o.l[0] = 1; return mul(a, o);
    }

    // a^(p-2); not on any per-element hot path (3 per proof + key precomputation)
    static __device__ __noinline__ fe inv(const fe& a) {
        const uint32_t e[8] = {P::P0 - 2u, P::P1, P::P2, P::P3, P::P4, P::P5, P::P6, P::P7};
        fe acc = one();
        for (int i = 255; i >= 0; i--) {
            acc = sqr(acc);
            if ((e[i >> 5] >> (i & 31)) & 1u) acc = mul(acc, a);
        }
        return acc;
    }

    // a^((p + 1) / 4), a square root of a whenever a has one (p = 3 mod 4: Fq only); is_root tells whether it is one.  The
    // exponent is (p >> 2) + 1, 252 bits of which 109 are set (Fq): 252 squarings and 109 products, about the cost of inv
    static __device__ __noinline__ fe sqrt(const fe& a, bool& is_root) {
        static_assert((P::P0 & 3u) == 3u, "sqrt needs p = 3 (mod 4)");
        const uint32_t e[8] = {(P::P0 >> 2 | P::P1 << 30) + 1u, P::P1 >> 2 | P::P2 << 30, P::P2 >> 2 | P::P3 << 30, P::P3 >> 2 | P::P4 << 30,
                               P::P4 >> 2 | P::P5 << 30, P::P5 >> 2 | P::P6 << 30, P::P6 >> 2 | P::P7 << 30, P::P7 >> 2};
        fe acc = one();
        for (int i = 251; i >= 0; i--) {
            acc = sqr(acc);
            if ((e[i >> 5] >> (i & 31)) & 1u) acc = mul(acc, a);
        }
        is_root = eq(sqr(acc), a);
        return acc;
    }
};

using Fq = Fp<FqParams>;
using Fr = Fp<FrParams>;

// ---------------------------------------------------------------------------------------------- Fq2 = Fq[u]/(u^2+1)
struct fe2 { fe c0, c1; };

// Fq2 mul / sqr / mul_sub are real calls for the kernels that use the generic Curve<Fq2> formulas (key-load tables, fold,
// reduce, glue): those are latency chains on few threads, and inlining every call multiplies their code size.  The G2
// accumulation kernel does not use them: it runs the lane-pair addition of ec.cuh on mul_inline / sqr_inline.
#define B2G_FQ2_CALL __noinline__
struct Fq2 {
    using elem = fe2;
    static __device__ __forceinline__ fe2 zero() { fe2 r; r.c0 = fe_zero(); r.c1 = fe_zero(); return r; }
    static __device__ __forceinline__ fe2 one() { fe2 r; r.c0 = Fq::one(); r.c1 = fe_zero(); return r; }
    static __device__ __forceinline__ bool is_zero(const fe2& a) { return fe_is_zero(a.c0) && fe_is_zero(a.c1); }
    static __device__ __forceinline__ bool eq(const fe2& a, const fe2& b) { return fe_equal(a.c0, b.c0) && fe_equal(a.c1, b.c1); }
    static __device__ __forceinline__ fe2 add(const fe2& a, const fe2& b) { fe2 r; r.c0 = Fq::add(a.c0, b.c0); r.c1 = Fq::add(a.c1, b.c1); return r; }
    static __device__ __forceinline__ fe2 sub(const fe2& a, const fe2& b) { fe2 r; r.c0 = Fq::sub(a.c0, b.c0); r.c1 = Fq::sub(a.c1, b.c1); return r; }
    static __device__ __forceinline__ fe2 dbl(const fe2& a) { fe2 r; r.c0 = Fq::dbl(a.c0); r.c1 = Fq::dbl(a.c1); return r; }
    static __device__ __forceinline__ fe2 neg(const fe2& a) { fe2 r; r.c0 = Fq::neg(a.c0); r.c1 = Fq::neg(a.c1); return r; }
    // Karatsuba over Fq2 with lazy reduction: three 512-bit products, two Montgomery reductions
    //   c0 = a0 b0 - a1 b1,  c1 = (a0 + a1)(b0 + b1) - a0 b0 - a1 b1
    // COLS picks the column form of the 512-bit products (Fq::mul_wide_cols) over the row form (Fq::mul_wide).
    template <bool COLS>
    static __device__ __forceinline__ fe2 karatsuba(const fe2& a, const fe2& b) {
        uint32_t v0[16], v1[16], v2[16];
        fe sa = add_noreduce(a.c0, a.c1), sb = add_noreduce(b.c0, b.c1);      // < 2p < 2^255
        if (COLS) {
            Fq::mul_wide_cols(v0, a.c0, b.c0);
            Fq::mul_wide_cols(v1, a.c1, b.c1);
            Fq::mul_wide_cols(v2, sa, sb);
        } else {
            Fq::mul_wide(v0, a.c0, b.c0);
            Fq::mul_wide(v1, a.c1, b.c1);
            Fq::mul_wide(v2, sa, sb);
        }
        Fq::sub_wide(v2, v0);
        Fq::sub_wide(v2, v1);                                                 // a0 b1 + a1 b0 in [0, 2 p^2)
        const uint32_t br = Fq::sub_wide(v0, v1);                             // a0 b0 - a1 b1 (mod 2^512)
        Fq::add_p_high(v0, br);                                               // + p * 2^256 if negative: now in [0, p^2) or [p R - p^2, p R)
        fe2 r; r.c0 = Fq::redc(v0); r.c1 = Fq::redc(v2);
        return r;
    }
    // the called form keeps the column products: no row-to-row dependency for the single-thread chains that call it
    static __device__ B2G_FQ2_CALL fe2 mul(const fe2& a, const fe2& b) { return karatsuba<true>(a, b); }
    // the inlined form uses the row products: 16 fewer live accumulator registers per product, which the lane-pair
    // accumulation needs to stay inside 128 registers (and it has four independent warps per scheduler to hide latency)
    static __device__ __forceinline__ fe2 mul_inline(const fe2& a, const fe2& b) { return karatsuba<false>(a, b); }
    static __device__ __forceinline__ fe add_noreduce(const fe& a, const fe& b) {
        fe s;
        asm("add.cc.u32 %0, %8, %16;\n\t"
            "addc.cc.u32 %1, %9, %17;\n\t"
            "addc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\t"
            "addc.cc.u32 %4, %12, %20;\n\t"
            "addc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\t"
            "addc.u32 %7, %15, %23;"
            : "=r"(s.l[0]), "=r"(s.l[1]), "=r"(s.l[2]), "=r"(s.l[3]), "=r"(s.l[4]), "=r"(s.l[5]), "=r"(s.l[6]), "=r"(s.l[7])
            : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
              "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
        return s;
    }
    // two calls rather than a fused a*b - c*d: only the glue kernels' handful of mixed additions use it (the G2 accumulation
    // computes the two products on the two lanes of a pair)
    static __device__ B2G_FQ2_CALL fe2 mul_sub(const fe2& a, const fe2& b, const fe2& c, const fe2& d) { return sub(mul(a, b), mul(c, d)); }
    // (a0 + a1 u)^2 = (a0 + a1)(a0 - a1) + 2 a0 a1 u: two Montgomery products
    static __device__ __forceinline__ fe2 sqr_inline(const fe2& a) {
        fe s = Fq::add(a.c0, a.c1), d = Fq::sub(a.c0, a.c1), m = Fq::mul(a.c0, a.c1);
        fe2 r; r.c0 = Fq::mul(s, d); r.c1 = Fq::dbl(m);
        return r;
    }
    static __device__ B2G_FQ2_CALL fe2 sqr(const fe2& a) { return sqr_inline(a); }
    // c ? a : b without a branch (SEL per limb)
    static __device__ __forceinline__ fe2 sel(bool c, const fe2& a, const fe2& b) {
        fe2 r;
        #pragma unroll
        for (int i = 0; i < 8; i++) { r.c0.l[i] = c ? a.c0.l[i] : b.c0.l[i]; r.c1.l[i] = c ? a.c1.l[i] : b.c1.l[i]; }
        return r;
    }
    // the value held by the other lane of an aligned lane pair (lanes 2k, 2k+1; `mask` names the pair)
    static __device__ __forceinline__ fe2 shfl_pair(unsigned mask, const fe2& a) {
        fe2 r;
        #pragma unroll
        for (int i = 0; i < 8; i++) { r.c0.l[i] = __shfl_xor_sync(mask, a.c0.l[i], 1); r.c1.l[i] = __shfl_xor_sync(mask, a.c1.l[i], 1); }
        return r;
    }
    static __device__ __noinline__ fe2 inv(const fe2& a) {
        fe d = Fq::inv(Fq::add(Fq::sqr(a.c0), Fq::sqr(a.c1)));
        fe2 r; r.c0 = Fq::mul(a.c0, d); r.c1 = Fq::neg(Fq::mul(a.c1, d));
        return r;
    }
    // a square root r of a by the norm method; false (r = 0) when a has none.  With delta = (a0 + sqrt(a0^2 + a1^2)) / 2
    // (delta = a0 when a1 = 0) and s = delta^((p + 1) / 4):
    //     s^2 = delta    ->  r = s + a1 / (2 s) u
    //     s^2 = -delta   ->  r = a1 / (2 s) + s u      (then (a0 - sqrt(norm)) / 2 = -a1^2 / (4 delta) is the residue)
    // so one exponentiation serves both candidates.  A non-residue norm means no root; the result is checked by squaring.
    // Cost: two Fq exponentiations (one when a1 = 0), one Fq inversion.
    static __device__ __noinline__ bool sqrt(fe2& r, const fe2& a) {
        r = zero();
        fe d = a.c0;
        bool direct;
        if (!fe_is_zero(a.c1)) {
            const fe alpha = Fq::sqrt(Fq::add(Fq::sqr(a.c0), Fq::sqr(a.c1)), direct);
            if (!direct) return false;
            fe half;                                                          // 1/2, Montgomery
            half.l[0] = 0x4f060572u; half.l[1] = 0x87bee7d2u; half.l[2] = 0x2f1c6ae5u; half.l[3] = 0xd0fd2addu;
            half.l[4] = 0xfcfd4f44u; half.l[5] = 0x8f5f7492u; half.l[6] = 0x3d9cbfacu; half.l[7] = 0x1f37631au;
            d = Fq::mul(Fq::add(a.c0, alpha), half);
        }
        const fe s = Fq::sqrt(d, direct);
        const fe t = Fq::mul(a.c1, Fq::inv(Fq::dbl(s)));
        fe2 c; c.c0 = direct ? s : t; c.c1 = direct ? t : s;
        if (!eq(sqr(c), a)) return false;
        r = c;
        return true;
    }
};

}  // namespace b2g
