// pairing.cuh - the BN254 optimal-ate pairing on the device: Fq6 / Fq12 tower, projective Miller loop, final exponentiation.
//
// Device counterpart of the host verifier's pairing (circom_compat_b200/verifier.py, host/ark_circom_verifier.hpp), on the
// same tower: u^2 = -1, v^3 = xi = 9 + u, w^2 = v.  An Fq12 is ((c0.c0, c0.c1, c0.c2), (c1.c0, c1.c1, c1.c2)) of Fq2, each
// Fq2 (c0, c1), twelve 32 B Montgomery residues in that order (384 B, the struct layout below).
//   - Miller loop over the signed digits of 6x + 2 (NAF, 22 nonzero digits against 37 set bits of the binary form) with
//     homogeneous projective line steps on the twist, so there is no inversion inside the loop; a line is the sparse
//     element c0 py + c1 px w + c2 w^3 (`mul_by_034`), then the two Frobenius lines pi(Q) and -pi^2(Q).  The projective
//     lines are the host's affine lines times a factor in Fq2, which the final exponentiation removes.
//   - Final exponentiation f^((p^12 - 1) / r), exactly: easy part conj(f) / f, then g^(p^2) g; hard part (p^4 - p^2 + 1) / r
//     as the exact decomposition in x and p of Scott et al. (three exp-by-x chains on Granger-Scott cyclotomic squarings,
//     Frobenius maps and a fixed product chain), so results equal the host's f^((p^12 - 1) / r) bit for bit.
// The constants below are pinned from the big-int model (`python -m oracle.pairing_model`); tests/test_pairing_model.py
// checks them against it.  Every product of the tower is a real call (Fq2::mul, and the Fq6 / Fq12 products here): one
// Fq12 is 192 registers, so the verifier's one-proof-per-thread kernels keep their tower values in local memory.
#pragma once
#include "ec.cuh"

namespace b2g {

struct fe6 { fe2 c0, c1, c2; };
struct fe12 { fe6 c0, c1; };

// ---------------------------------------------------------------------------------------------- pinned constants
// PAIRING_FROB[k - 1][e - 1] = xi^(e (p^k - 1) / 6), the factor of the coefficient at w^e under f -> f^(p^k), k = 1..3,
// e = 1..5 (c0.c0 -> w^0, c1.c0 -> w^1, c0.c1 -> w^2, c1.c1 -> w^3, c0.c2 -> w^4, c1.c2 -> w^5).  The twist Frobenius uses
// the same values: pi(x, y) = (conj(x) FROB[0][1], conj(y) FROB[0][2]), pi^2(x, y) = (x FROB[1][1], y FROB[1][2]).
__constant__ uint32_t PAIRING_FROB[3][5][16] = {
    {{0x33144907u, 0xaf9ba696u, 0x87afb78au, 0xca6b1d73u, 0xf08a2087u, 0x11bded5eu, 0x1a1f3a7cu, 0x02f34d75u, 0x4c492d72u, 0xa222ae23u, 0x565de15bu, 0xd00f02a4u, 0x53dfc926u, 0xdc2ff3a2u, 0xb3899551u, 0x10a75716u},
     {0x4563ab30u, 0xb5773b10u, 0xa9aa6454u, 0x347f91c8u, 0x242e0991u, 0x7a007127u, 0x118214ecu, 0x1956bcd8u, 0xa0aa4757u, 0x6e849f1eu, 0x89f89141u, 0xaa1c7b6du, 0xfae0ca3au, 0xb6e713cdu, 0x4e82ebc3u, 0x26694fbbu},
     {0x2936b629u, 0xe4bbdd0cu, 0xe133bacbu, 0xbb30f162u, 0xf9645366u, 0x31a9d1b6u, 0xa500f8ddu, 0x253570beu, 0x5ffe77c7u, 0xa1d77ce4u, 0x7826d1dbu, 0x07affd11u, 0xbb7edc6bu, 0x6d16bd27u, 0x85defeccu, 0x2c872002u},
     {0x843abe92u, 0x7361d77fu, 0x273411fbu, 0xa5bb2bd3u, 0x4b3e2399u, 0x9c941f31u, 0xbb9fd3ecu, 0x15df9cddu, 0x4bd8c949u, 0x5dddfd15u, 0xa4445b60u, 0x62cb29a5u, 0x0c7dd2b9u, 0x37bc870au, 0x3171f0fdu, 0x24830a9du},
     {0x41690fe7u, 0xc970692fu, 0x27694b0bu, 0xe2403421u, 0x83c459e8u, 0x32bee66bu, 0x0ab08841u, 0x12aabcedu, 0x40aebfa9u, 0x0d485d23u, 0xab2fcc57u, 0x05193418u, 0x8a4910f5u, 0xd3b0a40bu, 0x35d2925au, 0x2f21ebb5u}},
    {{0x00fa1bf2u, 0xca8d8005u, 0x68b39769u, 0xf0c5d614u, 0xad0d4418u, 0x0e201271u, 0xbad856e6u, 0x04290f65u, 0, 0, 0, 0, 0, 0, 0, 0},
     {0x13e80b9cu, 0x3350c88eu, 0xdb5e56b9u, 0x7dce557cu, 0xb615564au, 0x6001b4b8u, 0x020217e0u, 0x2682e617u, 0, 0, 0, 0, 0, 0, 0, 0},
     {0x12edefaau, 0x68c34889u, 0x72aabf4fu, 0x8d087f68u, 0x09081231u, 0x51e1a247u, 0x4729c0fau, 0x2259d6b1u, 0, 0, 0, 0, 0, 0, 0, 0},
     {0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du, 0, 0, 0, 0, 0, 0, 0, 0},
     {0xc494f1abu, 0x08cfc388u, 0x8d1373d4u, 0x19b31514u, 0xcb6c0213u, 0x584e90fdu, 0xdf2f8849u, 0x09e1685bu, 0, 0, 0, 0, 0, 0, 0, 0}},
    {{0x4e46d97du, 0x36531618u, 0xd4c96d9fu, 0x0af7129eu, 0xca1009b5u, 0x659da72fu, 0x83a20d23u, 0x08116d89u, 0xc39c1939u, 0xb1df4af7u, 0x8a73bf7fu, 0x3d9f0287u, 0x8caf0ae0u, 0x9b222092u, 0xeff054a6u, 0x26684515u},
     {0x16ad6badu, 0xc9af22f7u, 0x4aa662b2u, 0xb311782au, 0xe248c7f4u, 0x19eeaf64u, 0xe3439f82u, 0x20273e77u, 0xf7ce93acu, 0xacc02860u, 0x7ba76b4cu, 0x3933d581u, 0x446c8467u, 0x69e6188bu, 0x4417cc55u, 0x0a46036du},
     {0xaf46471eu, 0x5764af0au, 0x873e0fc1u, 0xdc50792eu, 0x881d04f6u, 0x86a673ffu, 0x3c30a74cu, 0x0b2eddb4u, 0x787e8580u, 0x9a490f32u, 0xf04af8b1u, 0x8fd16d7fu, 0xc6027bf2u, 0x4b39888eu, 0x5b52a15du, 0x03dd2e70u},
     {0x7b6762dfu, 0x448a93a5u, 0x28fdeadfu, 0xbfd62df5u, 0x0e9bd47au, 0xd858f5d0u, 0x3476ec58u, 0x06b03d4du, 0xbcc936d1u, 0x2b19daf4u, 0x56f4299fu, 0xa1a54e7au, 0x5adeaef1u, 0xb533eee0u, 0x84dda0b2u, 0x170c812bu},
     {0x75cf559fu, 0xe0bc4b22u, 0xc154e60fu, 0xc238b945u, 0x929a7d5eu, 0x803982a5u, 0xf7e4a37eu, 0x15ce052du, 0xbf3799a7u, 0x2d28efbdu, 0x1ad60773u, 0x9b097e3cu, 0xaf4a535bu, 0x982d4113u, 0xe3056063u, 0x24e18991u}}};
// 3 b' = 9 / (9 + u), the twist's curve constant times three (Montgomery c0 || c1), and 1/2 (Montgomery)
__constant__ uint32_t PAIRING_TWIST_B3[16] = {
    0xb62e0d6au, 0x3baa927cu, 0xd1b664fdu, 0xd71e7c52u, 0xd95d4664u, 0x03873e63u, 0x082ab8f4u, 0x0e75b5b1u,
    0x7596fe35u, 0xaab7c666u, 0xbb6a27bau, 0x31d21a78u, 0x680401ffu, 0x85dd7297u, 0xdf39a7e9u, 0x03c52d6au};
__constant__ uint32_t PAIRING_INV2[8] = {0x4f060572u, 0x87bee7d2u, 0x2f1c6ae5u, 0xd0fd2addu, 0xfcfd4f44u, 0x8f5f7492u, 0x3d9cbfacu, 0x1f37631au};
// 6x + 2 in non-adjacent form, most significant digit first, without its leading 1: one loop step per digit
constexpr int ATE_STEPS = 65;
__constant__ int8_t PAIRING_ATE_NAF[ATE_STEPS] = {
    0, -1, 0, 1, 0, 0, 0, -1, 0, -1, 0, 0, 0, -1, 0, 1, 0, -1, 0, 0, -1, 0, 0, 0, 0, 0, 1, 0, 0, -1, 0, 1, 0, 0, -1, 0, 0, 0, 0, -1, 0, 1, 0,
    0, 0, -1, 0, -1, 0, 0, 1, 0, 0, 0, -1, 0, 0, -1, 0, 1, 0, 1, 0, 0, 0};
// line steps of one G2 argument: one doubling per digit, one addition per nonzero digit, then the two Frobenius lines
constexpr int ATE_LINES = 65 + 21 + 2;
constexpr uint64_t PAIRING_X = 0x44e992b44a6909f1ull;                 // the BN parameter x (63 bits)
constexpr size_t LINE_BYTES = 3 * 64;                                 // (c0, c1, c2) Fq2 coefficients of one line

__device__ __forceinline__ fe const_fe(const uint32_t* w) { fe r; for (int i = 0; i < 8; i++) r.l[i] = w[i]; return r; }
__device__ __forceinline__ fe2 const_fe2(const uint32_t* w) { fe2 r; r.c0 = const_fe(w); r.c1 = const_fe(w + 8); return r; }
__device__ __forceinline__ fe2 frob_coeff(int k, int e) { return const_fe2(PAIRING_FROB[k - 1][e - 1]); }

// ---------------------------------------------------------------------------------------------- Fq2 helpers
__device__ __forceinline__ fe2 fq2_mul_xi(const fe2& a) {                 // (9 + u)(a0 + a1 u) = (9 a0 - a1) + (9 a1 + a0) u
    fe t0 = Fq::add(Fq::dbl(Fq::dbl(Fq::dbl(a.c0))), a.c0), t1 = Fq::add(Fq::dbl(Fq::dbl(Fq::dbl(a.c1))), a.c1);
    fe2 r; r.c0 = Fq::sub(t0, a.c1); r.c1 = Fq::add(t1, a.c0);
    return r;
}
__device__ __forceinline__ fe2 fq2_conj(const fe2& a) { fe2 r; r.c0 = a.c0; r.c1 = Fq::neg(a.c1); return r; }
__device__ __forceinline__ fe2 fq2_mul_fp(const fe2& a, const fe& k) { fe2 r; r.c0 = Fq::mul(a.c0, k); r.c1 = Fq::mul(a.c1, k); return r; }

// ---------------------------------------------------------------------------------------------- Fq6 = Fq2[v] / (v^3 - xi)
struct Fq6 {
    static __device__ __forceinline__ fe6 zero() { fe6 r; r.c0 = Fq2::zero(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
    static __device__ __forceinline__ fe6 add(const fe6& a, const fe6& b) { fe6 r; r.c0 = Fq2::add(a.c0, b.c0); r.c1 = Fq2::add(a.c1, b.c1); r.c2 = Fq2::add(a.c2, b.c2); return r; }
    static __device__ __forceinline__ fe6 sub(const fe6& a, const fe6& b) { fe6 r; r.c0 = Fq2::sub(a.c0, b.c0); r.c1 = Fq2::sub(a.c1, b.c1); r.c2 = Fq2::sub(a.c2, b.c2); return r; }
    static __device__ __forceinline__ fe6 neg(const fe6& a) { fe6 r; r.c0 = Fq2::neg(a.c0); r.c1 = Fq2::neg(a.c1); r.c2 = Fq2::neg(a.c2); return r; }
    static __device__ __forceinline__ fe6 mul_v(const fe6& a) { fe6 r; r.c0 = fq2_mul_xi(a.c2); r.c1 = a.c0; r.c2 = a.c1; return r; }

    // Karatsuba over Fq6: six Fq2 products
    static __device__ __noinline__ void mul(fe6& r, const fe6& a, const fe6& b) {
        const fe2 t0 = Fq2::mul(a.c0, b.c0), t1 = Fq2::mul(a.c1, b.c1), t2 = Fq2::mul(a.c2, b.c2);
        const fe2 m12 = Fq2::mul(Fq2::add(a.c1, a.c2), Fq2::add(b.c1, b.c2));
        const fe2 m01 = Fq2::mul(Fq2::add(a.c0, a.c1), Fq2::add(b.c0, b.c1));
        const fe2 m02 = Fq2::mul(Fq2::add(a.c0, a.c2), Fq2::add(b.c0, b.c2));
        r.c0 = Fq2::add(t0, fq2_mul_xi(Fq2::sub(Fq2::sub(m12, t1), t2)));
        r.c1 = Fq2::add(Fq2::sub(Fq2::sub(m01, t0), t1), fq2_mul_xi(t2));
        r.c2 = Fq2::add(Fq2::sub(Fq2::sub(m02, t0), t2), t1);
    }
    // a * (b0 + b1 v): five Fq2 products
    static __device__ __noinline__ void mul_by_01(fe6& r, const fe6& a, const fe2& b0, const fe2& b1) {
        const fe2 t0 = Fq2::mul(a.c0, b0), t1 = Fq2::mul(a.c1, b1);
        const fe2 m = Fq2::mul(Fq2::add(a.c0, a.c1), Fq2::add(b0, b1));
        const fe2 c0 = Fq2::add(fq2_mul_xi(Fq2::mul(a.c2, b1)), t0);
        const fe2 c2 = Fq2::add(Fq2::mul(a.c2, b0), t1);
        r.c1 = Fq2::sub(Fq2::sub(m, t0), t1);
        r.c0 = c0; r.c2 = c2;
    }
    static __device__ __noinline__ void inv(fe6& r, const fe6& a) {
        const fe2 c0 = Fq2::sub(Fq2::sqr(a.c0), fq2_mul_xi(Fq2::mul(a.c1, a.c2)));
        const fe2 c1 = Fq2::sub(fq2_mul_xi(Fq2::sqr(a.c2)), Fq2::mul(a.c0, a.c1));
        const fe2 c2 = Fq2::sub(Fq2::sqr(a.c1), Fq2::mul(a.c0, a.c2));
        const fe2 t = Fq2::inv(Fq2::add(Fq2::mul(a.c0, c0), fq2_mul_xi(Fq2::add(Fq2::mul(a.c2, c1), Fq2::mul(a.c1, c2)))));
        r.c0 = Fq2::mul(c0, t); r.c1 = Fq2::mul(c1, t); r.c2 = Fq2::mul(c2, t);
    }
};

// ---------------------------------------------------------------------------------------------- Fq12 = Fq6[w] / (w^2 - v)
struct Fq12 {
    static __device__ __forceinline__ fe12 one() { fe12 r; r.c0 = Fq6::zero(); r.c1 = Fq6::zero(); r.c0.c0 = Fq2::one(); return r; }
    static __device__ __forceinline__ bool eq(const fe12& a, const fe12& b) {
        return Fq2::eq(a.c0.c0, b.c0.c0) && Fq2::eq(a.c0.c1, b.c0.c1) && Fq2::eq(a.c0.c2, b.c0.c2) &&
               Fq2::eq(a.c1.c0, b.c1.c0) && Fq2::eq(a.c1.c1, b.c1.c1) && Fq2::eq(a.c1.c2, b.c1.c2);
    }
    static __device__ __forceinline__ fe12 conj(const fe12& a) { fe12 r; r.c0 = a.c0; r.c1 = Fq6::neg(a.c1); return r; }   // f^(p^6)
    static __device__ __forceinline__ fe12 load(const void* p) {
        fe12 r; fe2* e = &r.c0.c0;
        for (int i = 0; i < 6; i++) elem_load(e[i], (const char*)p + 64 * i);
        return r;
    }
    static __device__ __forceinline__ void store(void* p, const fe12& a) {
        const fe2* e = &a.c0.c0;
        for (int i = 0; i < 6; i++) elem_store((char*)p + 64 * i, e[i]);
    }

    // Karatsuba over Fq12: three Fq6 products (18 Fq2 products)
    static __device__ __noinline__ void mul(fe12& r, const fe12& a, const fe12& b) {
        fe6 t0, t1, m;
        Fq6::mul(t0, a.c0, b.c0);
        Fq6::mul(t1, a.c1, b.c1);
        Fq6::mul(m, Fq6::add(a.c0, a.c1), Fq6::add(b.c0, b.c1));
        r.c1 = Fq6::sub(Fq6::sub(m, t0), t1);
        r.c0 = Fq6::add(t0, Fq6::mul_v(t1));
    }
    // complex squaring: (a0 + a1 w)^2 = (a0 + a1)(a0 + v a1) - t - v t + 2 t w with t = a0 a1 (two Fq6 products)
    static __device__ __noinline__ void sqr(fe12& r, const fe12& a) {
        fe6 t, m;
        Fq6::mul(t, a.c0, a.c1);
        Fq6::mul(m, Fq6::add(a.c0, a.c1), Fq6::add(a.c0, Fq6::mul_v(a.c1)));
        r.c0 = Fq6::sub(Fq6::sub(m, t), Fq6::mul_v(t));
        r.c1 = Fq6::add(t, t);
    }
    // f * (c0 + c3 w + c4 w^3) for c0, c3, c4 in Fq2: the line as ((c0, 0, 0), (c3, c4, 0)), 13 Fq2 products
    static __device__ __noinline__ void mul_by_034(fe12& f, const fe2& c0, const fe2& c3, const fe2& c4) {
        fe6 a, b, m;
        a.c0 = Fq2::mul(f.c0.c0, c0); a.c1 = Fq2::mul(f.c0.c1, c0); a.c2 = Fq2::mul(f.c0.c2, c0);
        Fq6::mul_by_01(b, f.c1, c3, c4);
        Fq6::mul_by_01(m, Fq6::add(f.c0, f.c1), Fq2::add(c0, c3), c4);
        f.c1 = Fq6::sub(Fq6::sub(m, a), b);
        f.c0 = Fq6::add(a, Fq6::mul_v(b));
    }
    static __device__ __noinline__ void inv(fe12& r, const fe12& a) {
        fe6 t0, t1, t;
        Fq6::mul(t0, a.c0, a.c0);
        Fq6::mul(t1, a.c1, a.c1);
        Fq6::inv(t, Fq6::sub(t0, Fq6::mul_v(t1)));
        fe6 c1;
        Fq6::mul(c1, a.c1, t);
        Fq6::mul(r.c0, a.c0, t);
        r.c1 = Fq6::neg(c1);
    }
    // f^(p^k), k = 1, 2, 3: the coefficient at w^e becomes (conj if k is odd)(c) * PAIRING_FROB[k - 1][e - 1]
    static __device__ __noinline__ void frobenius(fe12& r, const fe12& a, int k) {
        const bool odd = k & 1;
        auto m = [&](const fe2& c) { return odd ? fq2_conj(c) : c; };
        r.c0.c0 = m(a.c0.c0);
        r.c1.c0 = Fq2::mul(m(a.c1.c0), frob_coeff(k, 1));
        r.c0.c1 = Fq2::mul(m(a.c0.c1), frob_coeff(k, 2));
        r.c1.c1 = Fq2::mul(m(a.c1.c1), frob_coeff(k, 3));
        r.c0.c2 = Fq2::mul(m(a.c0.c2), frob_coeff(k, 4));
        r.c1.c2 = Fq2::mul(m(a.c1.c2), frob_coeff(k, 5));
    }
    // Granger-Scott squaring in the cyclotomic subgroup: Fq12 as Fq4^3, Fq4 = Fq2[s] / (s^2 - xi), pairs (c0.c0, c1.c1),
    // (c1.c0, c0.c2), (c0.c1, c1.c2); three Fq4 squarings (six Fq2 products), then z -> 3 t -+ 2 z
    static __device__ __forceinline__ void fq4_sqr(fe2& r0, fe2& r1, const fe2& a, const fe2& b) {
        const fe2 t = Fq2::mul(a, b);
        r0 = Fq2::sub(Fq2::sub(Fq2::mul(Fq2::add(a, b), Fq2::add(a, fq2_mul_xi(b))), t), fq2_mul_xi(t));
        r1 = Fq2::dbl(t);
    }
    static __device__ __forceinline__ fe2 three_minus_two(const fe2& t, const fe2& z) { return Fq2::add(Fq2::dbl(Fq2::sub(t, z)), t); }
    static __device__ __forceinline__ fe2 three_plus_two(const fe2& t, const fe2& z) { return Fq2::add(Fq2::dbl(Fq2::add(t, z)), t); }
    static __device__ __noinline__ void cyclotomic_sqr(fe12& r, const fe12& a) {
        fe2 t0, t1, t2, t3, t4, t5;
        fq4_sqr(t0, t1, a.c0.c0, a.c1.c1);
        fq4_sqr(t2, t3, a.c1.c0, a.c0.c2);
        fq4_sqr(t4, t5, a.c0.c1, a.c1.c2);
        r.c0.c0 = three_minus_two(t0, a.c0.c0);
        r.c1.c1 = three_plus_two(t1, a.c1.c1);
        r.c1.c0 = three_plus_two(fq2_mul_xi(t5), a.c1.c0);
        r.c0.c2 = three_minus_two(t4, a.c0.c2);
        r.c0.c1 = three_minus_two(t2, a.c0.c1);
        r.c1.c2 = three_plus_two(t3, a.c1.c2);
    }
    // f^x for a cyclotomic f: 62 cyclotomic squarings and a product per set bit of x below its top bit
    static __device__ __noinline__ void exp_by_x(fe12& r, const fe12& f) {
        fe12 acc = f;
        #pragma unroll 1
        for (int i = 61; i >= 0; i--) {
            cyclotomic_sqr(acc, acc);
            if ((PAIRING_X >> i) & 1u) mul(acc, acc, f);
        }
        r = acc;
    }
    // f^k for a cyclotomic f and a canonical 256-bit k (8 x u32): square-and-multiply from the top set bit
    static __device__ __noinline__ void cyclotomic_exp(fe12& r, const fe12& f, const uint32_t* k) {
        int top = 255;
        while (top >= 0 && !((k[top >> 5] >> (top & 31)) & 1u)) top--;
        if (top < 0) { r = one(); return; }
        fe12 acc = f;
        #pragma unroll 1
        for (int i = top - 1; i >= 0; i--) {
            cyclotomic_sqr(acc, acc);
            if ((k[i >> 5] >> (i & 31)) & 1u) mul(acc, acc, f);
        }
        r = acc;
    }

    // f^((p^12 - 1) / r).  Hard part: with g cyclotomic and y0 = g^(p + p^2 + p^3), y1 = conj(g), y2 = (g^(x^2))^(p^2),
    // y3 = conj((g^x)^p), y4 = conj(g^x (g^(x^2))^p), y5 = conj(g^(x^2)), y6 = conj(g^(x^3) (g^(x^3))^p), the result is
    // y0 y1^2 y2^6 y3^12 y4^18 y5^30 y6^36 = g^((p^4 - p^2 + 1) / r) exactly (Scott et al., "On the final exponentiation for
    // calculating pairings on ordinary elliptic curves"), computed by a fixed chain of squarings and products.
    static __device__ __noinline__ void final_exponentiation(fe12& out, const fe12& f) {
        fe12 g, t, fx, fx2, fx3, y0, y3, y4, y6, t0, t1;
        inv(t, f);
        mul(g, conj(f), t);                                 // f^(p^6 - 1)
        frobenius(t, g, 2);
        mul(g, t, g);                                       // ^(p^2 + 1)
        exp_by_x(fx, g);
        exp_by_x(fx2, fx);
        exp_by_x(fx3, fx2);
        frobenius(t, g, 1); frobenius(y0, g, 2); mul(y0, t, y0); frobenius(t, g, 3); mul(y0, y0, t);
        frobenius(y3, fx, 1); y3 = conj(y3);
        frobenius(t, fx2, 1); mul(y4, fx, t); y4 = conj(y4);
        frobenius(t, fx3, 1); mul(y6, fx3, t); y6 = conj(y6);
        const fe12 y5 = conj(fx2);
        fe12 y2; frobenius(y2, fx2, 2);
        cyclotomic_sqr(t0, y6); mul(t0, t0, y4); mul(t0, t0, y5);
        mul(t1, y3, y5); mul(t1, t1, t0);
        mul(t0, t0, y2);
        cyclotomic_sqr(t1, t1); mul(t1, t1, t0);
        cyclotomic_sqr(t1, t1);
        mul(t0, t1, conj(g));                               // y1 = conj(g)
        mul(t1, t1, y0);
        cyclotomic_sqr(t0, t0);
        mul(out, t0, t1);
    }
};

// ---------------------------------------------------------------------------------------------- line steps on the twist
// T in homogeneous projective coordinates (x = X / Z, y = Y / Z) on E': y^2 = x^3 + b'.  A step returns the line's
// coefficients (c0, c1, c2); at the G1 point (px, py) the line is c0 py + c1 px w + c2 w^3.
struct G2Proj { fe2 x, y, z; };

// T = 2T; tangent (-2YZ, 3X^2, 3b'Z^2 - Y^2) = -2 y Z^2 times the affine tangent
__device__ __noinline__ void line_dbl(G2Proj& t, fe2* c) {
    const fe inv2 = const_fe(PAIRING_INV2);
    const fe2 a = fq2_mul_fp(Fq2::mul(t.x, t.y), inv2);
    const fe2 b = Fq2::sqr(t.y), cc = Fq2::sqr(t.z);
    const fe2 e = Fq2::mul(const_fe2(PAIRING_TWIST_B3), cc);
    const fe2 f = Fq2::add(Fq2::dbl(e), e);
    const fe2 g = fq2_mul_fp(Fq2::add(b, f), inv2);
    const fe2 h = Fq2::sub(Fq2::sqr(Fq2::add(t.y, t.z)), Fq2::add(b, cc));
    const fe2 j = Fq2::sqr(t.x);
    const fe2 e2 = Fq2::sqr(e);
    c[0] = Fq2::neg(h);
    c[1] = Fq2::add(Fq2::dbl(j), j);
    c[2] = Fq2::sub(e, b);
    t.x = Fq2::mul(a, Fq2::sub(b, f));
    t.y = Fq2::sub(Fq2::sqr(g), Fq2::add(Fq2::dbl(e2), e2));
    t.z = Fq2::mul(b, h);
}

// T = T + Q for affine Q; chord (X - qx Z, -(Y - qy Z), theta qx - lambda qy) = lambda times the affine chord
__device__ __noinline__ void line_add(G2Proj& t, const fe2& qx, const fe2& qy, fe2* c) {
    const fe2 theta = Fq2::sub(t.y, Fq2::mul(qy, t.z));
    const fe2 lambda = Fq2::sub(t.x, Fq2::mul(qx, t.z));
    const fe2 cc = Fq2::sqr(theta), d = Fq2::sqr(lambda);
    const fe2 e = Fq2::mul(lambda, d);
    const fe2 f = Fq2::mul(t.z, cc);
    const fe2 g = Fq2::mul(t.x, d);
    const fe2 h = Fq2::sub(Fq2::add(e, f), Fq2::dbl(g));
    c[0] = lambda;
    c[1] = Fq2::neg(theta);
    c[2] = Fq2::sub(Fq2::mul(theta, qx), Fq2::mul(lambda, qy));
    t.x = Fq2::mul(lambda, h);
    t.y = Fq2::sub(Fq2::mul(theta, Fq2::sub(g, h)), Fq2::mul(e, t.y));
    t.z = Fq2::mul(t.z, e);
}

// f *= the line c at (px, py)
__device__ __forceinline__ void ell(fe12& f, const fe2* c, const fe& px, const fe& py) {
    Fq12::mul_by_034(f, fq2_mul_fp(c[0], py), fq2_mul_fp(c[1], px), c[2]);
}

// pi(Q) and -pi^2(Q) on the twist
__device__ __forceinline__ void twist_frobenius(fe2& x1, fe2& y1, fe2& x2, fe2& y2, const fe2& qx, const fe2& qy) {
    x1 = Fq2::mul(fq2_conj(qx), frob_coeff(1, 2));
    y1 = Fq2::mul(fq2_conj(qy), frob_coeff(1, 3));
    x2 = Fq2::mul(qx, frob_coeff(2, 2));
    y2 = Fq2::neg(Fq2::mul(qy, frob_coeff(2, 3)));
}

// psi, the first map of twist_frobenius, on an XYZZ point: x = X / ZZ gives conj(x) FROB = conj(X) FROB / conj(ZZ)
__device__ __forceinline__ G2::Pt g2_psi(const G2::Pt& q) {
    G2::Pt r;
    r.x = Fq2::mul(fq2_conj(q.x), frob_coeff(1, 2));
    r.y = Fq2::mul(fq2_conj(q.y), frob_coeff(1, 3));
    r.zz = fq2_conj(q.zz);
    r.zzz = fq2_conj(q.zzz);
    return r;
}

// Q in G2, the order-r subgroup of the twist, for Q on the twist (infinity included):
//     [x + 1] Q + psi([x] Q) + psi^2([x] Q) == psi^3([2x] Q)
// (El Housni, Guillevic, Piellard, "Co-factor clearing and subgroup membership testing on pairing-friendly curves"), one
// 63-bit product instead of the 254-bit [r] Q
__device__ __noinline__ bool g2_in_subgroup(const G2::Aff& q) {
    if (G2::aff_is_inf(q)) return true;
    const uint32_t x[2] = {(uint32_t)PAIRING_X, (uint32_t)(PAIRING_X >> 32)};
    const G2::Pt xq = G2::mul_affine(q, x, 2);
    const G2::Pt p1 = g2_psi(xq);
    G2::Pt lhs = xq;
    G2::madd(lhs, q);
    G2::add(lhs, p1);
    G2::add(lhs, g2_psi(p1));
    return G2::pt_eq(lhs, g2_psi(g2_psi(g2_psi(G2::dbl(xq)))));
}

// The line sequence of a G2 argument Q (affine, not infinity), in loop order.  `emit(c)` receives each line; the prepared
// lines of a fixed argument and the variable argument of the Miller loop below walk the same sequence.
template <class Emit>
__device__ __forceinline__ void g2_line_walk(const fe2& qx, const fe2& qy, Emit&& emit) {
    G2Proj t; t.x = qx; t.y = qy; t.z = Fq2::one();
    const fe2 nqy = Fq2::neg(qy);
    fe2 c[3];
    #pragma unroll 1
    for (int k = 0; k < ATE_STEPS; k++) {
        line_dbl(t, c); emit(c);
        const int d = PAIRING_ATE_NAF[k];
        if (d) { line_add(t, qx, d > 0 ? qy : nqy, c); emit(c); }
    }
    fe2 x1, y1, x2, y2;
    twist_frobenius(x1, y1, x2, y2, qx, qy);
    line_add(t, x1, y1, c); emit(c);
    line_add(t, x2, y2, c); emit(c);
}

// f *= the prepared line `i` of each of the nfix fixed pairs (fp[j], lines[j]).  A real call: with this body inlined
// into the Miller loop, the loop produced values that differ from the model on sm_90a (CUDA 12.9); see miller_loop_t.
__device__ __noinline__ void ell_fixed(fe12& f, int i, int nfix, const Affine<Fq>* fp, const uint8_t* const* lines) {
    for (int j = 0; j < nfix; j++) {
        fe2 c[3];
        const uint8_t* l = lines[j] + (size_t)i * LINE_BYTES;
        elem_load_nc(c[0], l); elem_load_nc(c[1], l + 64); elem_load_nc(c[2], l + 128);
        ell(f, c, fp[j].x, fp[j].y);
    }
}

// Multi-Miller loop sharing one f: with V_ON, one pair (vp, vq) whose G2 point is stepped here, and NFIX pairs (fp[j],
// lines[j]) whose G2 lines were prepared (ATE_LINES x LINE_BYTES each).  Squaring happens before every step but the first
// (f = 1 there); every line of a step is multiplied in for all pairs.  The pair counts are template parameters: one
// specialised loop per shape keeps the absent pairs' code out of it.  A single loop taking the counts at run time, and
// this loop with ell_fixed inlined, both gave values that differ from the model on sm_90a (CUDA 12.9), while this form
// matches it bit for bit; the cause was not found.  Each kernel gets its own compiled copy of these calls, so the tests run
// the shipped kernels themselves: verify_miller_kernel (test op 49) and batch_pairs_kernel (op 53), tests/test_verify_stages.py.
template <bool V_ON, int NFIX>
__device__ __noinline__ void miller_loop_t(fe12& f, const Affine<Fq>& vp, const Affine<Fq2>& vq, const Affine<Fq>* fp,
                                           const uint8_t* const* lines) {
    fe12 acc = Fq12::one();
    int idx = 0;
    G2Proj t; t.x = vq.x; t.y = vq.y; t.z = Fq2::one();
    const fe2 nqy = Fq2::neg(vq.y);
    fe2 c[3];
    #pragma unroll 1
    for (int k = 0; k < ATE_STEPS; k++) {
        if (k) Fq12::sqr(acc, acc);
        if (V_ON) { line_dbl(t, c); ell(acc, c, vp.x, vp.y); }
        ell_fixed(acc, idx++, NFIX, fp, lines);
        const int d = PAIRING_ATE_NAF[k];
        if (d) {
            if (V_ON) { line_add(t, vq.x, d > 0 ? vq.y : nqy, c); ell(acc, c, vp.x, vp.y); }
            ell_fixed(acc, idx++, NFIX, fp, lines);
        }
    }
    if (V_ON) {
        fe2 x1, y1, x2, y2;
        twist_frobenius(x1, y1, x2, y2, vq.x, vq.y);
        line_add(t, x1, y1, c); ell(acc, c, vp.x, vp.y);
        ell_fixed(acc, idx++, NFIX, fp, lines);
        line_add(t, x2, y2, c); ell(acc, c, vp.x, vp.y);
        ell_fixed(acc, idx++, NFIX, fp, lines);
    } else {
        ell_fixed(acc, idx++, NFIX, fp, lines);
        ell_fixed(acc, idx++, NFIX, fp, lines);
    }
    f = acc;
}

// the loop for `v_on` (the stepped pair is present and not at infinity) and nfix (0..2) prepared pairs
__device__ __forceinline__ void miller_loop(fe12& f, bool v_on, const Affine<Fq>& vp, const Affine<Fq2>& vq, int nfix,
                                            const Affine<Fq>* fp, const uint8_t* const* lines) {
    if (v_on) {
        if (nfix == 0) miller_loop_t<true, 0>(f, vp, vq, fp, lines);
        else if (nfix == 1) miller_loop_t<true, 1>(f, vp, vq, fp, lines);
        else miller_loop_t<true, 2>(f, vp, vq, fp, lines);
    } else {
        if (nfix == 0) f = Fq12::one();
        else if (nfix == 1) miller_loop_t<false, 1>(f, vp, vq, fp, lines);
        else miller_loop_t<false, 2>(f, vp, vq, fp, lines);
    }
}

// e(P, Q) for affine points (Montgomery; infinity on either side gives 1)
__device__ __forceinline__ void pairing(fe12& out, const Affine<Fq>& p, const Affine<Fq2>& q) {
    fe12 f;
    miller_loop(f, !G1::aff_is_inf(p) && !G2::aff_is_inf(q), p, q, 0, nullptr, nullptr);
    Fq12::final_exponentiation(out, f);
}

}  // namespace b2g
