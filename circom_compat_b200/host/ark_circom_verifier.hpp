// ark_circom_verifier.hpp - Groth16 verification over BN254 on the host (C++ mirror of circom_compat_b200/verifier.py).
//
// Counterpart of the calls the reference makes right after proving (/root/reference/src/zkey.rs:868-870, 914-916;
// tests/groth16.rs:33-35):   GrothBn::process_vk(&params.vk)   and   GrothBn::verify_with_processed_vk(&pvk, &inputs, &proof).
// ark-groth16 0.5.0 semantics: prepared_inputs = gamma_abc_g1[0] + sum x_i gamma_abc_g1[i+1]; accept iff
//     e(A, B) * e(prepared_inputs, -gamma) * e(C, -delta) == e(alpha, beta);   MalformedVerifyingKey on an input-count mismatch.
// Milliseconds of host work, not part of the accelerated path.  Optimal ate pairing, Fq2 -> Fq6 -> Fq12 tower
// (u^2 = -1, v^3 = 9 + u, w^2 = v), affine line functions on the sextic D-twist, final exponent (p^6 - 1) * ((p^6 + 1) / r)
// by plain square-and-multiply.  Constants were produced by circom_compat_b200/verifier.py (xi^((p-1)/3) etc.).
// Included by ark_circom_b200.hpp (needs its Fr, G1Affine, G2Affine, VerifyingKey, Proof, detail::geq).
#pragma once

namespace ark_circom {

struct MalformedVerifyingKey : SynthesisError { MalformedVerifyingKey() : SynthesisError("MalformedVerifyingKey") {} };

namespace pairing {

// ------------------------------------------------------------------------------------------ Fq (4 x u64 Montgomery, R = 2^256)
static const uint64_t Q_INV = 0x87d20782e4866389ULL;
static const uint64_t Q_R2[4] = {0xf32cfc5b538afa89ULL, 0xb5e71911d44501fbULL, 0x47ab1eff0a417ff6ULL, 0x06d89f71cab8351fULL};
static const uint64_t Q_ONE[4] = {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL};

struct Fq {
    uint64_t l[4] = {0, 0, 0, 0};
    static Fq zero() { return Fq(); }
    static Fq one() { Fq f; memcpy(f.l, Q_ONE, 32); return f; }
    static Fq from_mont(const uint64_t* w) { Fq f; memcpy(f.l, w, 32); return f; }           // zkey / device layout
    static Fq from_canonical(const uint64_t* w) { Fq a, r2; memcpy(a.l, w, 32); memcpy(r2.l, Q_R2, 32); return a * r2; }
    static Fq from_u64(uint64_t v) { uint64_t w[4] = {v, 0, 0, 0}; return from_canonical(w); }
    bool is_zero() const { return !(l[0] | l[1] | l[2] | l[3]); }
    bool operator==(const Fq& o) const { return !memcmp(l, o.l, 32); }
    bool operator!=(const Fq& o) const { return !(*this == o); }
    Fq operator+(const Fq& o) const {
        Fq r; u128 c = 0;
        for (int i = 0; i < 4; i++) { c += (u128)l[i] + o.l[i]; r.l[i] = (uint64_t)c; c >>= 64; }
        if (detail::geq(r.l, detail::FQ_P)) r.sub_p();
        return r;
    }
    Fq operator-(const Fq& o) const {
        Fq r; uint64_t br = 0;
        for (int i = 0; i < 4; i++) { u128 d = (u128)l[i] - o.l[i] - br; r.l[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
        if (br) { u128 c = 0; for (int i = 0; i < 4; i++) { c += (u128)r.l[i] + detail::FQ_P[i]; r.l[i] = (uint64_t)c; c >>= 64; } }
        return r;
    }
    Fq operator-() const { return Fq() - *this; }
    Fq operator*(const Fq& o) const {
        uint64_t t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; i++) {
            u128 c = 0;
            for (int j = 0; j < 4; j++) { c += (u128)l[j] * o.l[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
            c += t[4]; t[4] = (uint64_t)c; t[5] = (uint64_t)(c >> 64);
            const uint64_t m = t[0] * Q_INV;
            c = (u128)m * detail::FQ_P[0] + t[0]; c >>= 64;
            for (int j = 1; j < 4; j++) { c += (u128)m * detail::FQ_P[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
            c += t[4]; t[3] = (uint64_t)c; c >>= 64;
            t[4] = t[5] + (uint64_t)c;
        }
        Fq r; memcpy(r.l, t, 32);
        if (t[4] || detail::geq(r.l, detail::FQ_P)) r.sub_p();
        return r;
    }
    Fq sqr() const { return *this * *this; }
    Fq dbl() const { return *this + *this; }
    Fq inv() const {                                                       // a^(p-2)
        uint64_t e[4]; memcpy(e, detail::FQ_P, 32); e[0] -= 2;
        Fq acc = one();
        for (int i = 255; i >= 0; i--) { acc = acc.sqr(); if ((e[i >> 6] >> (i & 63)) & 1) acc = acc * *this; }
        return acc;
    }
private:
    void sub_p() { uint64_t br = 0; for (int i = 0; i < 4; i++) { u128 d = (u128)l[i] - detail::FQ_P[i] - br; l[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; } }
};

// ------------------------------------------------------------------------------------------ the tower
struct Fq2 {
    Fq c0, c1;
    static Fq2 zero() { return Fq2(); }
    static Fq2 one() { Fq2 r; r.c0 = Fq::one(); return r; }
    bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
    Fq2 operator+(const Fq2& o) const { return {c0 + o.c0, c1 + o.c1}; }
    Fq2 operator-(const Fq2& o) const { return {c0 - o.c0, c1 - o.c1}; }
    Fq2 operator-() const { return {-c0, -c1}; }
    Fq2 operator*(const Fq2& o) const { Fq a = c0 * o.c0, b = c1 * o.c1; return {a - b, (c0 + c1) * (o.c0 + o.c1) - a - b}; }
    Fq2 sqr() const { Fq m = c0 * c1; return {(c0 + c1) * (c0 - c1), m + m}; }
    Fq2 scale(const Fq& k) const { return {c0 * k, c1 * k}; }
    Fq2 conj() const { return {c0, -c1}; }
    Fq2 mul_xi() const {                                                   // * (9 + u)
        Fq a8 = c0.dbl().dbl().dbl(), b8 = c1.dbl().dbl().dbl();
        return {a8 + c0 - c1, b8 + c1 + c0};
    }
    Fq2 inv() const { Fq d = (c0.sqr() + c1.sqr()).inv(); return {c0 * d, -(c1 * d)}; }
};

struct Fq6 {
    Fq2 c0, c1, c2;
    static Fq6 one() { Fq6 r; r.c0 = Fq2::one(); return r; }
    bool operator==(const Fq6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
    Fq6 operator+(const Fq6& o) const { return {c0 + o.c0, c1 + o.c1, c2 + o.c2}; }
    Fq6 operator-(const Fq6& o) const { return {c0 - o.c0, c1 - o.c1, c2 - o.c2}; }
    Fq6 operator-() const { return {-c0, -c1, -c2}; }
    Fq6 mul_v() const { return {c2.mul_xi(), c0, c1}; }
    Fq6 operator*(const Fq6& o) const {
        Fq2 t0 = c0 * o.c0, t1 = c1 * o.c1, t2 = c2 * o.c2;
        return {t0 + ((c1 + c2) * (o.c1 + o.c2) - t1 - t2).mul_xi(), (c0 + c1) * (o.c0 + o.c1) - t0 - t1 + t2.mul_xi(), (c0 + c2) * (o.c0 + o.c2) - t0 - t2 + t1};
    }
    Fq6 inv() const {
        Fq2 a = c0.sqr() - (c1 * c2).mul_xi(), b = c2.sqr().mul_xi() - c0 * c1, c = c1.sqr() - c0 * c2;
        Fq2 t = (c0 * a + (c2 * b + c1 * c).mul_xi()).inv();
        return {a * t, b * t, c * t};
    }
};

struct Fq12 {
    Fq6 c0, c1;
    static Fq12 one() { Fq12 r; r.c0 = Fq6::one(); return r; }
    bool operator==(const Fq12& o) const { return c0 == o.c0 && c1 == o.c1; }
    Fq12 operator*(const Fq12& o) const {
        Fq6 t0 = c0 * o.c0, t1 = c1 * o.c1;
        return {t0 + t1.mul_v(), (c0 + c1) * (o.c0 + o.c1) - t0 - t1};
    }
    Fq12 conj() const { return {c0, -c1}; }                                // p^6-power Frobenius
    Fq12 inv() const { Fq6 t = (c0 * c0 - (c1 * c1).mul_v()).inv(); return {c0 * t, -(c1 * t)}; }
    // f * (l0 + l1 w + l3 w^3): as a tower element ((l0, 0, 0), (l1, l3, 0))
    Fq12 mul_line(const Fq& l0, const Fq2& l1, const Fq2& l3) const {
        Fq12 l; l.c0.c0.c0 = l0; l.c1.c0 = l1; l.c1.c1 = l3;
        return *this * l;
    }
};

// ------------------------------------------------------------------------------------------ points (affine, flag = infinity)
struct P1 { Fq x, y; bool inf = true; };
struct P2 { Fq2 x, y; bool inf = true; };

inline P1 g1_from(const G1Affine& p) { P1 r; r.inf = p.is_infinity(); if (!r.inf) { r.x = Fq::from_mont(p.x); r.y = Fq::from_mont(p.y); } return r; }
inline P2 g2_from(const G2Affine& p) {
    P2 r; uint64_t o = 0; for (int i = 0; i < 4; i++) o |= p.x0[i] | p.x1[i] | p.y0[i] | p.y1[i];
    r.inf = !o;
    if (!r.inf) { r.x = {Fq::from_mont(p.x0), Fq::from_mont(p.x1)}; r.y = {Fq::from_mont(p.y0), Fq::from_mont(p.y1)}; }
    return r;
}
inline Fq2 twist_b() {                                                     // 3 / (9 + u)
    static const uint64_t b0[4] = {0x3267e6dc24a138e5ULL, 0xb5b4c5e559dbefa3ULL, 0x81be18991be06ac3ULL, 0x2b149d40ceb8aaaeULL};
    static const uint64_t b1[4] = {0xe4a2bd0685c315d2ULL, 0xa74fa084e52d1852ULL, 0xcd2cafadeed8fdf4ULL, 0x009713b03af0fed4ULL};
    return {Fq::from_canonical(b0), Fq::from_canonical(b1)};
}
inline bool on_curve(const P1& p) { return p.inf || p.y.sqr() == p.x.sqr() * p.x + Fq::from_u64(3); }
inline bool on_curve(const P2& p) { return p.inf || p.y.sqr() == p.x.sqr() * p.x + twist_b(); }

inline P1 g1_add(const P1& a, const P1& b) {
    if (a.inf) return b;
    if (b.inf) return a;
    Fq lam;
    if (a.x == b.x) {
        if ((a.y + b.y).is_zero()) return P1();
        Fq xx = a.x.sqr();
        lam = (xx + xx + xx) * a.y.dbl().inv();
    } else lam = (b.y - a.y) * (b.x - a.x).inv();
    P1 r; r.inf = false;
    r.x = lam.sqr() - a.x - b.x;
    r.y = lam * (a.x - r.x) - a.y;
    return r;
}
inline P1 g1_mul(P1 p, const BigInt256& k) {                               // canonical scalar
    P1 acc;
    for (int i = 0; i < 256; i++) {
        if ((k.l[i >> 6] >> (i & 63)) & 1) acc = g1_add(acc, p);
        p = g1_add(p, p);
    }
    return acc;
}
inline P2 g2_neg(const P2& p) { P2 r = p; if (!r.inf) r.y = -r.y; return r; }

// ------------------------------------------------------------------------------------------ optimal ate pairing
// line through t and q (tangent when equal) on the twist evaluated at (xp, yp); t <- t + q.  Untwisting (x', y') ->
// (x' w^2, y' w^3) turns the slope lambda into lambda w:  l(P) = yp - (lambda xp) w + (lambda x_t - y_t) w^3
inline void line_step(Fq12& f, P2& t, const P2& q, const Fq& xp, const Fq& yp) {
    Fq2 lam;
    if (t.x == q.x && t.y == q.y) { Fq2 xx = t.x.sqr(); lam = (xx + xx + xx) * (t.y + t.y).inv(); }
    else lam = (q.y - t.y) * (q.x - t.x).inv();
    Fq2 x3 = lam.sqr() - t.x - q.x;
    Fq2 y3 = lam * (t.x - x3) - t.y;
    f = f.mul_line(yp, lam.scale(-xp), lam * t.x - t.y);
    t.x = x3; t.y = y3;
}

inline Fq12 miller_loop(const std::vector<std::pair<P1, P2>>& in) {
    // xi^((p-1)/3), xi^((p-1)/2), xi^((p^2-1)/3), xi^((p^2-1)/2)  (canonical; the last two lie in Fq)
    static const uint64_t G12[2][4] = {{0x99e39557176f553dULL, 0xb78cc310c2c3330cULL, 0x4c0bec3cf559b143ULL, 0x2fb347984f7911f7ULL},
                                       {0x1665d51c640fcba2ULL, 0x32ae2a1d0b7c9dceULL, 0x4ba4cc8bd75a0794ULL, 0x16c9e55061ebae20ULL}};
    static const uint64_t G13[2][4] = {{0xdc54014671a0135aULL, 0xdbaae0eda9c95998ULL, 0xdc5ec698b6e2f9b9ULL, 0x063cf305489af5dcULL},
                                       {0x82d37f632623b0e3ULL, 0x21807dc98fa25bd2ULL, 0x0704b5a7ec796f2bULL, 0x07c03cbcac41049aULL}};
    static const uint64_t G22[4] = {0xe4bd44e5607cfd48ULL, 0xc28f069fbb966e3dULL, 0x5e6dd9e7e0acccb0ULL, 0x30644e72e131a029ULL};
    static const uint64_t G23[4] = {0x3c208c16d87cfd46ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
    const Fq2 g12 = {Fq::from_canonical(G12[0]), Fq::from_canonical(G12[1])}, g13 = {Fq::from_canonical(G13[0]), Fq::from_canonical(G13[1])};
    const Fq g22 = Fq::from_canonical(G22), g23 = Fq::from_canonical(G23);
    std::vector<std::pair<P1, P2>> pairs;
    for (const auto& pq : in) if (!pq.first.inf && !pq.second.inf) pairs.push_back(pq);        // infinity contributes 1
    std::vector<P2> ts;
    for (const auto& pq : pairs) ts.push_back(pq.second);
    Fq12 f = Fq12::one();
    const unsigned __int128 loop = ((unsigned __int128)0x1ULL << 64) | 0x9d797039be763ba8ULL;  // 6x + 2 = 29793968203157093288
    for (int i = 63; i >= 0; i--) {
        f = f * f;
        for (size_t k = 0; k < pairs.size(); k++) { P2 t = ts[k]; line_step(f, ts[k], t, pairs[k].first.x, pairs[k].first.y); }
        if ((loop >> i) & 1) for (size_t k = 0; k < pairs.size(); k++) line_step(f, ts[k], pairs[k].second, pairs[k].first.x, pairs[k].first.y);
    }
    for (size_t k = 0; k < pairs.size(); k++) {
        const P2& q = pairs[k].second;
        P2 q1; q1.inf = false; q1.x = q.x.conj() * g12; q1.y = q.y.conj() * g13;               // pi(Q)
        P2 q2; q2.inf = false; q2.x = q.x.scale(g22); q2.y = -(q.y.scale(g23));                // -pi^2(Q)
        line_step(f, ts[k], q1, pairs[k].first.x, pairs[k].first.y);
        line_step(f, ts[k], q2, pairs[k].first.x, pairs[k].first.y);
    }
    return f;
}

inline Fq12 final_exponentiation(const Fq12& f) {
    // (p^6 + 1) / r, little-endian limbs (1268 bits)
    static const uint64_t E[20] = {0x5250a54036e3f812ULL, 0xa5635f1596789051ULL, 0xd1138bf54d5bd1d4ULL, 0xa8ce2533be36c7a2ULL, 0x94f69f6b84e09bf6ULL,
                                   0x42ad1f5e50ef3644ULL, 0x0fcc420e48c3454cULL, 0x758e4408ecc9952cULL, 0xc901bf1887c6042cULL, 0xa733cd65b14bb3b5ULL,
                                   0xdf6d76bdcf51b0d8ULL, 0xca64c0fd82eb59e1ULL, 0x1d2e5726e39276a1ULL, 0xc2d1ea74a391cae9ULL, 0x07409206c82d647eULL,
                                   0x051c6d1aa5afdd17ULL, 0xb37f601919667af5ULL, 0x150e578c5084015bULL, 0xfbdea556c23998e4ULL, 0x000fd14cc52f5b83ULL};
    const Fq12 g = f.conj() * f.inv();                                     // f^(p^6 - 1)
    Fq12 acc = Fq12::one();
    for (int i = 1267; i >= 0; i--) { acc = acc * acc; if ((E[i >> 6] >> (i & 63)) & 1) acc = acc * g; }
    return acc;
}

}  // namespace pairing

// PreparedVerifyingKey<Bn254> (ark-groth16 prepare_verifying_key): vk, e(alpha, beta), -gamma, -delta
struct PreparedVerifyingKey {
    VerifyingKey vk;
    pairing::Fq12 alpha_g1_beta_g2;
    pairing::P2 gamma_g2_neg, delta_g2_neg;
    DeviceSlot device;                                  // the key prepared on a device (b2g_vk_load) by Groth16::verify_many
    void release_device() const { device.release(); }
};

inline PreparedVerifyingKey prepare_verifying_key(const VerifyingKey& vk) {
    using namespace pairing;
    PreparedVerifyingKey p; p.vk = vk;
    P1 alpha = g1_from(vk.alpha_g1); P2 beta = g2_from(vk.beta_g2), gamma = g2_from(vk.gamma_g2), delta = g2_from(vk.delta_g2);
    if (!on_curve(alpha) || !on_curve(beta) || !on_curve(gamma) || !on_curve(delta)) throw SerializationError("verifying key point not on the curve");
    for (const auto& ic : vk.gamma_abc_g1) if (!on_curve(g1_from(ic))) throw SerializationError("verifying key point not on the curve");
    p.alpha_g1_beta_g2 = final_exponentiation(miller_loop({{alpha, beta}}));
    p.gamma_g2_neg = g2_neg(gamma); p.delta_g2_neg = g2_neg(delta);
    return p;
}

// proof bytes = canonical little-endian coordinates (struct Proof); all-zero coordinates = infinity
inline bool verify_with_processed_vk(const PreparedVerifyingKey& pvk, const std::vector<Fr>& public_inputs, const Proof& proof) {
    using namespace pairing;
    if (public_inputs.size() + 1 != pvk.vk.gamma_abc_g1.size()) throw MalformedVerifyingKey();
    auto coord = [&](int slot) { uint64_t w[4]; memcpy(w, proof.bytes + 32 * slot, 32); if (detail::geq(w, detail::FQ_P)) throw SerializationError("proof coordinate not reduced"); return w[0] | w[1] | w[2] | w[3] ? Fq::from_canonical(w) : Fq::zero(); };
    P1 a, c; P2 b;
    a.x = coord(0); a.y = coord(1); a.inf = a.x.is_zero() && a.y.is_zero();
    b.x = {coord(2), coord(3)}; b.y = {coord(4), coord(5)}; b.inf = b.x.is_zero() && b.y.is_zero();
    c.x = coord(6); c.y = coord(7); c.inf = c.x.is_zero() && c.y.is_zero();
    if (!on_curve(a) || !on_curve(b) || !on_curve(c)) return false;
    P1 acc = g1_from(pvk.vk.gamma_abc_g1[0]);
    for (size_t i = 0; i < public_inputs.size(); i++) acc = g1_add(acc, g1_mul(g1_from(pvk.vk.gamma_abc_g1[i + 1]), public_inputs[i].into_bigint()));
    Fq12 f = miller_loop({{a, b}, {acc, pvk.gamma_g2_neg}, {c, pvk.delta_g2_neg}});
    return final_exponentiation(f) == pvk.alpha_g1_beta_g2;
}

}  // namespace ark_circom
