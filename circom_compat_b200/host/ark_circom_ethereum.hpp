// ark_circom_ethereum.hpp - Ethereum-facing views of a proof and a verifying key (C++ mirror of circom_compat_b200/ethereum.py).
//
// Counterpart of /root/reference/src/ethereum.rs: `Inputs` (:10-18), `G1` (:20-54), `G2` (:56-95; as_tuple emits c1 BEFORE
// c0, :82-86), `Proof` (:98-128), `VerifyingKey` (:130-174), `u256_to_point` / `point_to_u256` (:176-189), in both directions
// like the reference (`From<&G1Affine> for G1` and `From<G1> for G1Affine`, ...).  A U256 is the canonical integer of a
// coordinate as 32 big-endian bytes (what `U256::from(&bytes_be[..])` holds and what the Solidity verifier of
// tests/solidity.rs receives).  The point at infinity is (0, 0), as in the reference (:26-39, :61-80).
// ark_circom::serialize_compressed mirrors ethereum.py's encoder of arkworks' 128-byte compressed proof.
// Host-side formatting of a handful of points; included by ark_circom_b200.hpp after the verifier (needs pairing::Fq).
#pragma once

#include <array>

namespace ark_circom {
namespace ethereum {

struct U256 {
    uint8_t be[32];
    bool operator==(const U256& o) const { return !memcmp(be, o.be, 32); }
    bool is_zero() const { for (uint8_t b : be) if (b) return false; return true; }
    std::string hex() const { static const char* d = "0123456789abcdef"; std::string s; for (uint8_t b : be) { s += d[b >> 4]; s += d[b & 15]; } return s; }
};

namespace detail_eth {
inline U256 from_canonical_limbs(const uint64_t w[4]) {
    U256 u;
    for (int i = 0; i < 4; i++) for (int k = 0; k < 8; k++) u.be[31 - (8 * i + k)] = (uint8_t)(w[i] >> (8 * k));
    return u;
}
inline void to_canonical_limbs(const U256& u, uint64_t w[4]) {
    for (int i = 0; i < 4; i++) { w[i] = 0; for (int k = 0; k < 8; k++) w[i] |= (uint64_t)u.be[31 - (8 * i + k)] << (8 * k); }
}
}  // namespace detail_eth

// point_to_u256 (src/ethereum.rs:185-189) for a base-field coordinate held as Montgomery limbs (the zkey / device layout)
inline U256 fq_to_u256(const uint64_t mont[4]) {
    pairing::Fq one_raw; one_raw.l[0] = 1;                                  // a * 1 * R^-1 = the canonical integer
    const pairing::Fq c = pairing::Fq::from_mont(mont) * one_raw;
    return detail_eth::from_canonical_limbs(c.l);
}
// u256_to_point (src/ethereum.rs:176-181): `F::from_bigint(..).expect(..)` panics on a value >= q; here it throws
inline void u256_to_fq(const U256& u, uint64_t mont_out[4]) {
    uint64_t w[4]; detail_eth::to_canonical_limbs(u, w);
    if (detail::geq(w, detail::FQ_P)) throw SerializationError("U256 is not a canonical Fq element");
    const pairing::Fq m = pairing::Fq::from_canonical(w);
    memcpy(mont_out, m.l, 32);
}
inline U256 fr_to_u256(const Fr& x) { const BigInt256 b = x.into_bigint(); return detail_eth::from_canonical_limbs(b.l); }
inline Fr u256_to_fr(const U256& u) { BigInt256 b; detail_eth::to_canonical_limbs(u, b.l); return Fr::from_bigint(b); }   // throws if >= r

// Inputs(Vec<U256>) from &[Fr] (src/ethereum.rs:10-18)
inline std::vector<U256> inputs(const std::vector<Fr>& public_inputs) {
    std::vector<U256> v; v.reserve(public_inputs.size());
    for (const Fr& x : public_inputs) v.push_back(fr_to_u256(x));
    return v;
}

struct G1 {
    U256 x, y;
    static G1 from(const G1Affine& p) {                                     // From<&G1Affine> for G1 (:46-54); infinity -> (0, 0)
        G1 g; memset(&g, 0, sizeof g);
        if (!p.is_infinity()) { g.x = fq_to_u256(p.x); g.y = fq_to_u256(p.y); }
        return g;
    }
    G1Affine into() const {                                                 // From<G1> for G1Affine (:26-39)
        G1Affine p; memset(&p, 0, sizeof p);
        if (!(x.is_zero() && y.is_zero())) { u256_to_fq(x, p.x); u256_to_fq(y, p.y); }
        return p;
    }
    std::array<U256, 2> as_tuple() const { return {x, y}; }
    bool operator==(const G1& o) const { return x == o.x && y == o.y; }
};

struct G2 {
    U256 x[2], y[2];                                                        // [c0, c1]
    static G2 from(const G2Affine& p) {                                     // From<&G2Affine> for G2 (:88-95)
        G2 g; memset(&g, 0, sizeof g);
        uint64_t o = 0; for (int i = 0; i < 4; i++) o |= p.x0[i] | p.x1[i] | p.y0[i] | p.y1[i];
        if (o) { g.x[0] = fq_to_u256(p.x0); g.x[1] = fq_to_u256(p.x1); g.y[0] = fq_to_u256(p.y0); g.y[1] = fq_to_u256(p.y1); }
        return g;
    }
    G2Affine into() const {                                                 // From<G2> for G2Affine (:61-80)
        G2Affine p; memset(&p, 0, sizeof p);
        if (!(x[0].is_zero() && x[1].is_zero() && y[0].is_zero() && y[1].is_zero())) {
            u256_to_fq(x[0], p.x0); u256_to_fq(x[1], p.x1); u256_to_fq(y[0], p.y0); u256_to_fq(y[1], p.y1);
        }
        return p;
    }
    // ([x.c1, x.c0], [y.c1, y.c0]): c1 first (src/ethereum.rs:82-86)
    std::array<std::array<U256, 2>, 2> as_tuple() const { return {{{x[1], x[0]}, {y[1], y[0]}}}; }
    bool operator==(const G2& o) const { return x[0] == o.x[0] && x[1] == o.x[1] && y[0] == o.y[0] && y[1] == o.y[1]; }
};

// Proof (src/ethereum.rs:98-128).  ark_circom::Proof holds canonical LITTLE-endian coordinates, so the conversion is a byte swap.
struct Proof {
    G1 a; G2 b; G1 c;
    static Proof from(const ark_circom::Proof& p) {
        auto word = [&](int slot) { U256 u; for (int k = 0; k < 32; k++) u.be[31 - k] = p.bytes[32 * slot + k]; return u; };
        Proof e;
        e.a.x = word(0); e.a.y = word(1);
        e.b.x[0] = word(2); e.b.x[1] = word(3); e.b.y[0] = word(4); e.b.y[1] = word(5);
        e.c.x = word(6); e.c.y = word(7);
        return e;
    }
    ark_circom::Proof into() const {
        ark_circom::Proof p;
        const U256* w[8] = {&a.x, &a.y, &b.x[0], &b.x[1], &b.y[0], &b.y[1], &c.x, &c.y};
        for (int s = 0; s < 8; s++) {
            uint64_t limbs[4]; detail_eth::to_canonical_limbs(*w[s], limbs);
            if (detail::geq(limbs, detail::FQ_P)) throw SerializationError("U256 is not a canonical Fq element");
            for (int k = 0; k < 32; k++) p.bytes[32 * s + k] = w[s]->be[31 - k];
        }
        return p;
    }
    // abi.encode(uint[2] a, uint[2][2] b, uint[2] c): the eight words in the order the Solidity verifier takes them
    std::array<U256, 8> calldata_words() const { const auto bt = b.as_tuple(); return {a.x, a.y, bt[0][0], bt[0][1], bt[1][0], bt[1][1], c.x, c.y}; }
    bool operator==(const Proof& o) const { return a == o.a && b == o.b && c == o.c; }
};

// VerifyingKey (src/ethereum.rs:130-174)
struct VerifyingKey {
    G1 alpha1; G2 beta2, gamma2, delta2; std::vector<G1> ic;
    static VerifyingKey from(const ark_circom::VerifyingKey& vk) {
        VerifyingKey e;
        e.alpha1 = G1::from(vk.alpha_g1); e.beta2 = G2::from(vk.beta_g2); e.gamma2 = G2::from(vk.gamma_g2); e.delta2 = G2::from(vk.delta_g2);
        for (const G1Affine& p : vk.gamma_abc_g1) e.ic.push_back(G1::from(p));
        return e;
    }
    ark_circom::VerifyingKey into() const {
        ark_circom::VerifyingKey vk;
        vk.alpha_g1 = alpha1.into(); vk.beta_g2 = beta2.into(); vk.gamma_g2 = gamma2.into(); vk.delta_g2 = delta2.into();
        for (const G1& p : ic) vk.gamma_abc_g1.push_back(p.into());
        return vk;
    }
};

}  // namespace ethereum

// ---------------------------------------------------------------------------------------------- ark-serialize
// Proof::<Bn254>::serialize_compressed (ark-serialize 0.5, restated like ethereum.py's serialize_compressed, byte for byte
// equal to it): A.x (32 B), B.x.c0, B.x.c1, C.x, little-endian; the flags of each point ride in the top two bits of its last
// byte: bit 6 = infinity, bit 7 = y is the larger of {y, -y} (Fq2: c1 compared first, then c0).
typedef std::array<uint8_t, 128> CompressedProof;

namespace detail_eth {
// canonical little-endian coordinate y (32 B) against p - y (0 for y = 0): -1, 0 or 1
inline int cmp_neg(const uint8_t* yb) {
    uint64_t y[4], n[4] = {0, 0, 0, 0};
    memcpy(y, yb, 32);
    if (y[0] | y[1] | y[2] | y[3]) {
        unsigned __int128 br = 0;
        for (int i = 0; i < 4; i++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[i] - y[i] - (uint64_t)br; n[i] = (uint64_t)t; br = (t >> 64) & 1; }
    }
    for (int i = 3; i >= 0; i--) if (y[i] != n[i]) return y[i] > n[i] ? 1 : -1;
    return 0;
}
inline bool all_zero(const uint8_t* b, size_t n) { for (size_t i = 0; i < n; i++) if (b[i]) return false; return true; }
}  // namespace detail_eth

inline CompressedProof serialize_compressed(const Proof& p) {
    CompressedProof out;
    const uint8_t* b = p.bytes;
    auto g1 = [&](uint8_t* o, const uint8_t* xy) {
        memcpy(o, xy, 32);
        o[31] |= detail_eth::all_zero(xy, 64) ? 0x40 : (detail_eth::cmp_neg(xy + 32) > 0 ? 0x80 : 0);
    };
    g1(out.data(), b);
    memcpy(out.data() + 32, b + 64, 64);                                   // B.x.c0, B.x.c1
    const int c1 = detail_eth::cmp_neg(b + 160);
    out[95] |= detail_eth::all_zero(b + 64, 128) ? 0x40 : ((c1 ? c1 : detail_eth::cmp_neg(b + 128)) > 0 ? 0x80 : 0);
    g1(out.data() + 96, b + 192);
    return out;
}

}  // namespace ark_circom
