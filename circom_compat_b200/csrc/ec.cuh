// ec.cuh - BN254 G1 / G2 group arithmetic on the device (y^2 = x^3 + b, a = 0), templated over the coordinate field.
//
// Device-side counterpart of what ark-ec 0.5.0 does for the reference's prover (bucket `+=` affine, running sums,
// doublings; SURVEY.md App. C.3).  Buckets use extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ,
// ZZ^3 = ZZZ^2): a mixed addition is 8M+2S and needs no inversion; infinity is ZZ == 0.  Affine points use the zkey
// convention (/root/reference/src/zkey.rs:340-360): x||y Montgomery, all-zero = infinity.
#pragma once
#include "fp.cuh"

namespace b2g {

template <class F>
struct Affine { typename F::elem x, y; };

template <class F>
struct XYZZ { typename F::elem x, y, zz, zzz; };

template <class F>
struct Curve {
    using E = typename F::elem;
    using Aff = Affine<F>;
    using Pt = XYZZ<F>;

    static __device__ __forceinline__ bool aff_is_inf(const Aff& p) { return F::is_zero(p.x) && F::is_zero(p.y); }
    static __device__ __forceinline__ bool is_inf(const Pt& p) { return F::is_zero(p.zz); }
    static __device__ __forceinline__ Pt infinity() { Pt r; r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero(); return r; }
    static __device__ __forceinline__ Pt from_affine(const Aff& p) {
        Pt r;
        if (aff_is_inf(p)) return infinity();
        r.x = p.x; r.y = p.y; r.zz = F::one(); r.zzz = F::one();
        return r;
    }
    static __device__ __forceinline__ Pt neg(const Pt& p) { Pt r = p; r.y = F::neg(p.y); return r; }

    // 2*(x, y) for an affine, non-infinity point (mdbl-2008-s-1)
    static __device__ __forceinline__ Pt dbl_affine(const Aff& p) {
        Pt r;
        E u = F::dbl(p.y);
        E v = F::sqr(u);
        E w = F::mul(u, v);
        E s = F::mul(p.x, v);
        E xx = F::sqr(p.x);
        E m = F::add(F::dbl(xx), xx);
        r.x = F::sub(F::sqr(m), F::dbl(s));
        r.y = F::sub(F::mul(m, F::sub(s, r.x)), F::mul(w, p.y));
        r.zz = v; r.zzz = w;
        return r;
    }

    // 2*p (dbl-2008-s-1); y == 0 cannot happen on a prime-order curve except at infinity
    static __device__ __forceinline__ Pt dbl(const Pt& p) {
        if (is_inf(p)) return p;
        Pt r;
        E u = F::dbl(p.y);
        E v = F::sqr(u);
        E w = F::mul(u, v);
        E s = F::mul(p.x, v);
        E xx = F::sqr(p.x);
        E m = F::add(F::dbl(xx), xx);
        r.x = F::sub(F::sqr(m), F::dbl(s));
        r.y = F::sub(F::mul(m, F::sub(s, r.x)), F::mul(w, p.y));
        r.zz = F::mul(v, p.zz);
        r.zzz = F::mul(w, p.zzz);
        return r;
    }

    // acc += q (mixed addition madd-2008-s), every exceptional case handled
    static __device__ __forceinline__ void madd(Pt& acc, const Aff& q) {
        if (aff_is_inf(q)) return;
        if (is_inf(acc)) { acc.x = q.x; acc.y = q.y; acc.zz = F::one(); acc.zzz = F::one(); return; }
        E u2 = F::mul(q.x, acc.zz);
        E s2 = F::mul(q.y, acc.zzz);
        E p = F::sub(u2, acc.x);
        E r = F::sub(s2, acc.y);
        if (F::is_zero(p)) {
            if (F::is_zero(r)) acc = dbl_affine(q);
            else acc = infinity();
            return;
        }
        E pp = F::sqr(p);
        E ppp = F::mul(p, pp);
        E qq = F::mul(acc.x, pp);
        E x3 = F::sub(F::sub(F::sqr(r), ppp), F::dbl(qq));
        E y3 = F::mul_sub(r, F::sub(qq, x3), acc.y, ppp);
        acc.x = x3; acc.y = y3;
        acc.zz = F::mul(acc.zz, pp);
        acc.zzz = F::mul(acc.zzz, ppp);
    }

    // acc += q (add-2008-s)
    static __device__ __forceinline__ void add(Pt& acc, const Pt& q) {
        if (is_inf(q)) return;
        if (is_inf(acc)) { acc = q; return; }
        E u1 = F::mul(acc.x, q.zz);
        E u2 = F::mul(q.x, acc.zz);
        E s1 = F::mul(acc.y, q.zzz);
        E s2 = F::mul(q.y, acc.zzz);
        E p = F::sub(u2, u1);
        E r = F::sub(s2, s1);
        if (F::is_zero(p)) {
            if (F::is_zero(r)) acc = dbl(acc);
            else acc = infinity();
            return;
        }
        E pp = F::sqr(p);
        E ppp = F::mul(p, pp);
        E qq = F::mul(u1, pp);
        E x3 = F::sub(F::sub(F::sqr(r), ppp), F::dbl(qq));
        E y3 = F::sub(F::mul(r, F::sub(qq, x3)), F::mul(s1, ppp));
        acc.x = x3; acc.y = y3;
        acc.zz = F::mul(F::mul(acc.zz, q.zz), pp);
        acc.zzz = F::mul(F::mul(acc.zzz, q.zzz), ppp);
    }

    // k * p for a canonical 256-bit scalar (8 x u32), plain double-and-add from the top set bit
    static __device__ __noinline__ Pt mul_scalar(const Pt& p, const uint32_t* k) {
        Pt acc = infinity();
        int top = 255;
        while (top >= 0 && !((k[top >> 5] >> (top & 31)) & 1u)) top--;
        for (int i = top; i >= 0; i--) {
            acc = dbl(acc);
            if ((k[i >> 5] >> (i & 31)) & 1u) add(acc, p);
        }
        return acc;
    }

    // k * p for an affine p and a short scalar of `words` x u32 (little-endian): double-and-add over every bit with mixed
    // additions (the batch verifier's 128-bit weights, the G2 subgroup check's 63-bit x)
    static __device__ __noinline__ Pt mul_affine(const Aff& p, const uint32_t* k, int words) {
        Pt acc = infinity();
        #pragma unroll 1
        for (int i = 32 * words - 1; i >= 0; i--) {
            acc = dbl(acc);
            if ((k[i >> 5] >> (i & 31)) & 1u) madd(acc, p);
        }
        return acc;
    }

    // the same point: X1 ZZ2 == X2 ZZ1 and Y1 ZZZ2 == Y2 ZZZ1, or both at infinity
    static __device__ __forceinline__ bool pt_eq(const Pt& a, const Pt& b) {
        if (is_inf(a) || is_inf(b)) return is_inf(a) && is_inf(b);
        return F::eq(F::mul(a.x, b.zz), F::mul(b.x, a.zz)) && F::eq(F::mul(a.y, b.zzz), F::mul(b.y, a.zzz));
    }

    // XYZZ -> affine (Montgomery); infinity -> zeros.  One inversion: iz = 1/ZZZ, 1/ZZ = ZZ^2 * iz^2.
    static __device__ __noinline__ Aff to_affine(const Pt& p) {
        Aff r;
        if (is_inf(p)) { r.x = F::zero(); r.y = F::zero(); return r; }
        E iz = F::inv(p.zzz);
        r.y = F::mul(p.y, iz);
        E izz = F::mul(F::sqr(p.zz), F::sqr(iz));
        r.x = F::mul(p.x, izz);
        return r;
    }
};

using G1 = Curve<Fq>;
using G2 = Curve<Fq2>;

// ---------------------------------------------------------------------------------------------- G2 on a lane pair
// Two adjacent lanes (2k = A, 2k+1 = B) hold one XYZZ accumulator between them and split the ten Fq2 products of the mixed
// addition 5 / 5 by role, running the same instruction sequence on lane-selected operands:
//   lane A holds (X, ZZ) and the table point's x:   U2 = x2 ZZ1,   PP = P^2,  Q = X1 PP,    ZZ3 = ZZ1 PP,    R (Q - X3)
//   lane B holds (Y, ZZZ) and the table point's y:  S2 = y2 ZZZ1,  RR = R^2,  PPP = P PP,   ZZZ3 = ZZZ1 PPP, Y1 PPP
// Intermediates cross by __shfl_xor_sync(pair, ., 1); every branch is taken on values both lanes hold, so a pair never
// diverges.  `s0` / `s1` are the lane's two coordinates (A: X, ZZ; B: Y, ZZZ) - the halves of the 256 B XYZZ record each
// lane loads and stores - and `empty` (identical on both lanes) marks the accumulator at infinity (s0 = s1 = 0).
struct G2Pair {
    // acc = 2 q for the affine point q (mdbl-2008-s-1); `qc` is the lane's coordinate of q (A: x, B: y)
    static __device__ __forceinline__ void dbl_affine(fe2& s0, fe2& s1, const fe2& qc, bool A, unsigned mask) {
        const fe2 o1 = Fq2::sel(A, qc, Fq2::dbl(qc));                     // A: x,  B: U = 2y
        const fe2 sq = Fq2::sqr_inline(o1), sq_o = Fq2::shfl_pair(mask, sq); // A: XX, B: V = U^2
        const fe2 v = Fq2::sel(A, sq_o, sq), xx = Fq2::sel(A, sq, sq_o);
        const fe2 m2 = Fq2::mul_inline(o1, v), m2_o = Fq2::shfl_pair(mask, m2);    // A: S = x V, B: W = U V
        const fe2 s = Fq2::sel(A, m2, m2_o), w = Fq2::sel(A, m2_o, m2);
        const fe2 m = Fq2::add(Fq2::dbl(xx), xx);
        const fe2 x3 = Fq2::sub(Fq2::sqr_inline(m), Fq2::dbl(s));
        const fe2 m4 = Fq2::mul_inline(Fq2::sel(A, m, w), Fq2::sel(A, Fq2::sub(s, x3), qc));   // A: M (S - X3), B: W y
        const fe2 m4_o = Fq2::shfl_pair(mask, m4);
        s0 = Fq2::sel(A, x3, Fq2::sub(m4_o, m4));
        s1 = Fq2::sel(A, v, w);
    }

    // acc += q (madd-2008-s), every exceptional case handled; `qc` is the lane's coordinate of q (A: x, B: y)
    static __device__ __forceinline__ void madd(fe2& s0, fe2& s1, bool& empty, const fe2& qc, bool A, unsigned mask) {
        const bool qz = Fq2::is_zero(qc);
        const bool qz_o = __shfl_xor_sync(mask, (int)qz, 1) != 0;
        if (qz && qz_o) return;                                               // q at infinity
        if (empty) { s0 = qc; s1 = Fq2::one(); empty = false; return; }
        const fe2 d = Fq2::sub(Fq2::mul_inline(qc, s1), s0);                  // A: P = U2 - X1, B: R = S2 - Y1
        const fe2 d_o = Fq2::shfl_pair(mask, d);
        const bool z = Fq2::is_zero(d), z_o = Fq2::is_zero(d_o);
        if (A ? z : z_o) {                                                    // P == 0: q == acc (R == 0) or q == -acc
            if (A ? z_o : z) dbl_affine(s0, s1, qc, A, mask);
            else { s0 = Fq2::zero(); s1 = Fq2::zero(); empty = true; }
            return;
        }
        const fe2 u = Fq2::sel(A, s0, d_o);                                   // A: X1, B: P
        const fe2 v = Fq2::sel(A, d_o, s0);                                   // A: R,  B: Y1
        const fe2 sq = Fq2::sqr_inline(d);                                    // A: PP, B: RR
        const fe2 pp = Fq2::sel(A, sq, Fq2::shfl_pair(mask, sq));
        const fe2 m3 = Fq2::mul_inline(u, pp);                                // A: Q,  B: PPP
        const fe2 rp = Fq2::shfl_pair(mask, Fq2::sub(sq, m3));                // A receives RR - PPP
        const fe2 x3 = Fq2::sub(rp, Fq2::dbl(m3));                            // A: X3 = RR - PPP - 2Q
        const fe2 b5 = Fq2::sel(A, Fq2::sub(m3, x3), m3);                     // A: Q - X3, B: PPP
        s1 = Fq2::mul_inline(s1, Fq2::sel(A, pp, m3));                        // A: ZZ3 = ZZ1 PP, B: ZZZ3 = ZZZ1 PPP
        const fe2 m5 = Fq2::mul_inline(v, b5);                                // A: R (Q - X3), B: Y1 PPP
        const fe2 m5_o = Fq2::shfl_pair(mask, m5);
        s0 = Fq2::sel(A, x3, Fq2::sub(m5_o, m5));                             // B: Y3 = R (Q - X3) - Y1 PPP
    }
};

// curve constants b (y^2 = x^3 + b): G1 b = 3, G2 b = 3 / (9 + u)   (SURVEY.md App. A)
__device__ __forceinline__ fe curve_b(const Fq*) { fe t = fe_zero(); t.l[0] = 3; return Fq::from_canonical(t); }
__device__ __forceinline__ fe2 curve_b(const Fq2*) {
    fe c0, c1;
    c0.l[0] = 0x24a138e5u; c0.l[1] = 0x3267e6dcu; c0.l[2] = 0x59dbefa3u; c0.l[3] = 0xb5b4c5e5u; c0.l[4] = 0x1be06ac3u; c0.l[5] = 0x81be1899u; c0.l[6] = 0xceb8aaaeu; c0.l[7] = 0x2b149d40u;
    c1.l[0] = 0x85c315d2u; c1.l[1] = 0xe4a2bd06u; c1.l[2] = 0xe52d1852u; c1.l[3] = 0xa74fa084u; c1.l[4] = 0xeed8fdf4u; c1.l[5] = 0xcd2cafadu; c1.l[6] = 0x3af0fed4u; c1.l[7] = 0x009713b0u;
    fe2 r; r.c0 = Fq::from_canonical(c0); r.c1 = Fq::from_canonical(c1);
    return r;
}
// on-curve test of an affine point (infinity = all zero is accepted): the check G1Affine::new / G2Affine::new performs
// when the reference parses a zkey (/root/reference/src/zkey.rs:340-360, panics if it fails)
template <class C, class F>
__device__ __forceinline__ bool aff_on_curve(const Affine<F>& p) {
    if (C::aff_is_inf(p)) return true;
    typename F::elem lhs = F::sqr(p.y);
    typename F::elem rhs = F::add(F::mul(F::sqr(p.x), p.x), curve_b((const F*)nullptr));
    return F::eq(lhs, rhs);
}

// ---------------------------------------------------------------------------------------------- memory layout helpers
// G1 affine = 64 B (x||y), G2 affine = 128 B (x.c0||x.c1||y.c0||y.c1); XYZZ = 4 coordinates back to back.
__device__ __forceinline__ void elem_load(fe& r, const void* p) { r = fe_load(p); }
__device__ __forceinline__ void elem_load(fe2& r, const void* p) { r.c0 = fe_load(p); r.c1 = fe_load((const char*)p + 32); }
__device__ __forceinline__ void elem_load_nc(fe& r, const void* p) { r = fe_load_nc(p); }
__device__ __forceinline__ void elem_load_nc(fe2& r, const void* p) { r.c0 = fe_load_nc(p); r.c1 = fe_load_nc((const char*)p + 32); }
__device__ __forceinline__ void elem_store(void* p, const fe& v) { fe_store(p, v); }
__device__ __forceinline__ void elem_store(void* p, const fe2& v) { fe_store(p, v.c0); fe_store((char*)p + 32, v.c1); }

template <class F> struct Bytes;
template <> struct Bytes<Fq> { static constexpr int ELEM = 32; };
template <> struct Bytes<Fq2> { static constexpr int ELEM = 64; };

template <class F>
__device__ __forceinline__ Affine<F> aff_load(const void* base, size_t idx) {
    const char* p = (const char*)base + idx * (2 * Bytes<F>::ELEM);
    Affine<F> r; elem_load_nc(r.x, p); elem_load_nc(r.y, p + Bytes<F>::ELEM);
    return r;
}
template <class F>
__device__ __forceinline__ void aff_store(void* base, size_t idx, const Affine<F>& v) {
    char* p = (char*)base + idx * (2 * Bytes<F>::ELEM);
    elem_store(p, v.x); elem_store(p + Bytes<F>::ELEM, v.y);
}
template <class F>
__device__ __forceinline__ XYZZ<F> pt_load(const void* base, size_t idx) {
    const char* p = (const char*)base + idx * (4 * Bytes<F>::ELEM);
    XYZZ<F> r; elem_load(r.x, p); elem_load(r.y, p + Bytes<F>::ELEM); elem_load(r.zz, p + 2 * Bytes<F>::ELEM); elem_load(r.zzz, p + 3 * Bytes<F>::ELEM);
    return r;
}
template <class F>
__device__ __forceinline__ void pt_store(void* base, size_t idx, const XYZZ<F>& v) {
    char* p = (char*)base + idx * (4 * Bytes<F>::ELEM);
    elem_store(p, v.x); elem_store(p + Bytes<F>::ELEM, v.y); elem_store(p + 2 * Bytes<F>::ELEM, v.zz); elem_store(p + 3 * Bytes<F>::ELEM, v.zzz);
}

}  // namespace b2g
