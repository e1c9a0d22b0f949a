// ark_circom_b200.hpp - C++ host-side mirror of the ark-circom proving interface, on top of the C ABI (include/b2groth.h).
//
// The reference is compiled Rust and no Rust toolchain exists in the build image, so the host layer a user links
// against is C++ with the reference's names, argument meaning and error behaviour:
//
//   ark_circom::read_zkey(reader)                      <- /root/reference/src/zkey.rs:53-60 (+ BinFile :73-133, :151-196)
//   ark_circom::ProvingKey / ConstraintMatrices        <- ProvingKey<Bn254> (zkey.rs:121-130) / ConstraintMatrices<Fr> (zkey.rs:181-193)
//   ark_circom::CircomReduction::witness_map_from_matrices      <- src/circom/qap.rs:23-88
//   ark_circom::Groth16::create_proof_with_reduction_and_matrices <- call sites src/zkey.rs:903-912, benches/groth16.rs:52-61
//   ark_circom::Groth16::prove                         <- src/zkey.rs:866 (draws r then s, SURVEY.md App. C.5)
//   ark_circom::Groth16::process_vk / verify_with_processed_vk / verify <- src/zkey.rs:868-870, tests/groth16.rs:33-35
//   ark_circom::Groth16::verify_many          <- verify_with_processed_vk for many proofs of one key, in one device pass
//                                                         (host pairing, ark_circom_verifier.hpp; no GPU involved)
//   ark_circom::Groth16::verify_batch         <- the same for a whole batch at once: one random-linear-combination check
//   ark_circom::Groth16::decompress_proofs    <- Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5) for many proofs
//   ark_circom::Groth16::verify_many_compressed / verify_batch_compressed <- deserialize_compressed, then the two above
//   ark_circom::Groth16::verify_batch_keys (+ _compressed) <- verify_batch for many keys in one device pass, a verdict per key
//   ark_circom::Groth16::verify_batch_keys_locate (+ _compressed) <- verify_batch_locate for many keys in one device pass, a
//                             verdict per proof
//   ark_circom::Groth16::verify_batch_locate (+ _compressed) <- verify_with_processed_vk for every proof, at about the batch
//                                              check's cost when few proofs are invalid
//   ark_circom::Groth16::rerandomize_proof / rerandomize_many <- Groth16::rerandomize_proof (ark-groth16 0.5.0), many
//                                              proofs of one key in one device pass
//   ark_circom::serialize_compressed          <- Proof::<Bn254>::serialize_compressed (ark_circom_ethereum.hpp)
//   ark_circom::serialize_proving_key / deserialize_proving_key / serialize_verifying_key / deserialize_verifying_key(s)
//                                             <- CanonicalSerialize / CanonicalDeserialize (ark-serialize 0.5, Validate::Yes)
//                                                of ProvingKey<Bn254> / VerifyingKey<Bn254>, points decoded on the device
//   ark_circom::read_ptau + Groth16::generate_parameters_from_powers_of_tau <- snarkjs groth16 setup (a key from a ceremony)
//   ark_circom::Groth16::contribute / verify_contribution <- snarkjs zkey contribute / the delta checks of snarkjs zkey verify
//   ark_circom::Groth16::verify_powers_of_tau <- the algebraic checks of snarkjs powersoftau verify
//   ark_circom::Groth16::verify_proving_key <- snarkjs zkey verify: a key against its circuit and ceremony
//   ark_circom::read_wtns                              <- snarkjs .wtns (test-vectors/circuit2_js/witness.wtns; the reference
//                                                         computes witnesses with WASM instead, out of scope here)
// Parsing and key handling stay on the host; every field/curve operation of the proof runs in libb2groth.so.
// Header-only; link with -lb2groth.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <exception>
#include <fstream>
#include <istream>
#include <iterator>
#include <map>
#include <memory>
#include <optional>
#include <random>
#include <sstream>
#include <type_traits>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/b2groth.h"

namespace ark_circom {

// ---------------------------------------------------------------------------------------------- errors
struct SerializationError : std::runtime_error { using std::runtime_error::runtime_error; };                 // zkey.rs:43
struct SynthesisError : std::runtime_error { using std::runtime_error::runtime_error; };
struct PolynomialDegreeTooLarge : SynthesisError { PolynomialDegreeTooLarge() : SynthesisError("PolynomialDegreeTooLarge") {} };  // qap.rs:31
struct DeviceError : std::runtime_error { using std::runtime_error::runtime_error; };

inline void check(int rc) {
    if (rc == B2G_OK) return;
    if (rc == B2G_E_DOMAIN) throw PolynomialDegreeTooLarge();
    throw DeviceError(std::string("b2groth error ") + std::to_string(rc) + ": " + b2g_last_error());
}

// ---------------------------------------------------------------------------------------------- Fr (host side: conversions only)
typedef unsigned __int128 u128;
struct BigInt256 { uint64_t l[4]; };

namespace detail {
static const uint64_t FR_P[4] = {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
static const uint64_t FQ_P[4] = {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
static const uint64_t FR_INV = 0xc2e1f593efffffffULL;
static const uint64_t FR_R2[4] = {0x1bb8e645ae216da7ULL, 0x53fe3ab1e35c59e3ULL, 0x8c49833d53bb8085ULL, 0x0216d0b17f4e44a5ULL};

inline bool geq(const uint64_t a[4], const uint64_t p[4]) {
    for (int i = 3; i >= 0; i--) { if (a[i] > p[i]) return true; if (a[i] < p[i]) return false; }
    return true;
}
// Montgomery product mod r (host, used for encodings only - never for the proof)
inline void fr_mont_mul(uint64_t out[4], const uint64_t a[4], const uint64_t b[4]) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        u128 c = 0;
        for (int j = 0; j < 4; j++) { c += (u128)a[j] * b[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[4] = (uint64_t)c; t[5] = (uint64_t)(c >> 64);
        uint64_t m = t[0] * FR_INV;
        c = (u128)m * FR_P[0] + t[0]; c >>= 64;
        for (int j = 1; j < 4; j++) { c += (u128)m * FR_P[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[3] = (uint64_t)c; c >>= 64;
        t[4] = t[5] + (uint64_t)c;
    }
    if (t[4] || geq(t, FR_P)) { u128 br = 0; for (int i = 0; i < 4; i++) { u128 d = (u128)t[i] - FR_P[i] - (uint64_t)br; t[i] = (uint64_t)d; br = (d >> 64) & 1; } }
    memcpy(out, t, 32);
}
}  // namespace detail

// Fr as arkworks keeps it: 4 x u64 Montgomery limbs (Fp256<MontBackend>)
struct Fr {
    uint64_t l[4] = {0, 0, 0, 0};
    static Fr new_unchecked(const BigInt256& b) { Fr f; memcpy(f.l, b.l, 32); return f; }          // limbs ARE the residue
    static Fr from_bigint(const BigInt256& b) {                                                     // canonical -> Montgomery
        if (detail::geq(b.l, detail::FR_P)) throw std::invalid_argument("Fr::from_bigint: not reduced");
        Fr f; detail::fr_mont_mul(f.l, b.l, detail::FR_R2); return f;
    }
    static Fr from_u64(uint64_t v) { BigInt256 b = {{v, 0, 0, 0}}; return from_bigint(b); }
    BigInt256 into_bigint() const { const uint64_t one[4] = {1, 0, 0, 0}; BigInt256 b; detail::fr_mont_mul(b.l, l, one); return b; }
    bool is_zero() const { return !(l[0] | l[1] | l[2] | l[3]); }
    bool operator==(const Fr& o) const { return !memcmp(l, o.l, 32); }
    // Fr::rand of ark-ff 0.5 (SURVEY.md App. C.5): 4 limbs from the rng, top two bits cleared, rejected if >= r,
    // interpreted as the Montgomery residue
    template <class Rng> static Fr rand(Rng& rng) {
        for (;;) {
            BigInt256 b;
            for (int i = 0; i < 4; i++) b.l[i] = rng();
            b.l[3] &= 0x3fffffffffffffffULL;
            if (!detail::geq(b.l, detail::FR_P)) return new_unchecked(b);
        }
    }
};

struct G1Affine { uint64_t x[4], y[4]; bool is_infinity() const { uint64_t o = 0; for (int i = 0; i < 4; i++) o |= x[i] | y[i]; return !o; } };   // Montgomery, zeros = infinity
struct G2Affine { uint64_t x0[4], x1[4], y0[4], y1[4]; };
static_assert(sizeof(G1Affine) == 64 && sizeof(G2Affine) == 128, "zkey point layout");

struct VerifyingKey { G1Affine alpha_g1; G2Affine beta_g2, gamma_g2, delta_g2; std::vector<G1Affine> gamma_abc_g1; };

// Device copies (fixed-base tables, CSR matrices) belong to the host object they were made from: the slot is a member
// of ProvingKey / ConstraintMatrices, so the gigabytes of HBM are freed when that object dies, and a copy or an
// assignment - the ways a *different* key can come to live at the same address - start with an empty slot.  The device
// copy is a snapshot taken at first use: after mutating a key in place call release_device().
class DeviceSlot {
public:
    DeviceSlot() = default;
    DeviceSlot(const DeviceSlot&) {}                                   // a copy has no device state of its own yet
    DeviceSlot(DeviceSlot&& o) noexcept : handles_(std::move(o.handles_)), free_(o.free_) { o.handles_.clear(); }
    DeviceSlot& operator=(const DeviceSlot&) { release(); return *this; }   // new contents => stale tables must go
    DeviceSlot& operator=(DeviceSlot&& o) noexcept { if (this != &o) { release(); handles_ = std::move(o.handles_); free_ = o.free_; o.handles_.clear(); } return *this; }
    ~DeviceSlot() { release(); }
    void release() const { for (auto& kv : handles_) if (kv.second && free_) free_(kv.second); handles_.clear(); }
    void* find(const void* ctx, uint32_t tag) const { auto it = handles_.find({ctx, tag}); return it == handles_.end() ? nullptr : it->second; }
    void put(const void* ctx, uint32_t tag, void* h, void (*free_fn)(void*)) const { handles_[{ctx, tag}] = h; free_ = free_fn; }
private:
    mutable std::map<std::pair<const void*, uint32_t>, void*> handles_;       // (b2g_ctx, variant) -> b2g_pk* / b2g_mat*
    mutable void (*free_)(void*) = nullptr;
};

struct ProvingKey {                                     // ProvingKey<Bn254>, src/zkey.rs:121-130
    VerifyingKey vk;
    G1Affine beta_g1, delta_g1;
    std::vector<G1Affine> a_query, b_g1_query, h_query, l_query;
    std::vector<G2Affine> b_g2_query;
    DeviceSlot device;                                  // see DeviceSlot
    void release_device() const { device.release(); }
};

typedef std::vector<std::vector<std::pair<Fr, size_t>>> Matrix;     // rows of (coeff, index): src/zkey.rs:168

struct ConstraintMatrices {                             // src/zkey.rs:181-193
    size_t num_instance_variables = 0, num_witness_variables = 0, num_constraints = 0;
    size_t a_num_non_zero = 0, b_num_non_zero = 0, c_num_non_zero = 0;
    Matrix a, b, c;
    DeviceSlot device;
    void release_device() const { device.release(); }
};

struct Proof {                                          // Proof<Bn254>; coordinates canonical little-endian
    uint8_t bytes[256];                                 // A.x A.y B.x.c0 B.x.c1 B.y.c0 B.y.c1 C.x C.y
    std::string hex() const { static const char* d = "0123456789abcdef"; std::string s; for (uint8_t b : bytes) { s += d[b >> 4]; s += d[b & 15]; } return s; }
};

// ---------------------------------------------------------------------------------------------- zkey reader (host)
namespace detail {
struct Section { uint64_t position, size; };
inline void read_exact(std::istream& r, void* dst, size_t n) {
    r.read(reinterpret_cast<char*>(dst), (std::streamsize)n);
    if ((size_t)r.gcount() != n) throw SerializationError("unexpected end of zkey");
}
template <class T> inline T read_le(std::istream& r) { T v; read_exact(r, &v, sizeof(T)); return v; }   // x86: little-endian host
}  // namespace detail

class BinFile {                                         // src/zkey.rs:62-101
public:
    explicit BinFile(std::istream& reader) : r_(reader) {
        char magic[4]; detail::read_exact(r_, magic, 4);
        ftype_.assign(magic, 4);
        version_ = detail::read_le<uint32_t>(r_);
        uint32_t nsec = detail::read_le<uint32_t>(r_);
        for (uint32_t i = 0; i < nsec; i++) {
            uint32_t id = detail::read_le<uint32_t>(r_);
            uint64_t len = detail::read_le<uint64_t>(r_);
            sections_[id].push_back({(uint64_t)r_.tellg(), len});
            r_.seekg((std::streamoff)len, std::ios::cur);
            if (!r_) throw SerializationError("truncated zkey section table");
        }
        if (ftype_ != "zkey") throw SerializationError("not a zkey file");
    }

    ProvingKey proving_key() {                          // src/zkey.rs:103-133
        Header h = groth_header();
        ProvingKey pk;
        pk.vk.alpha_g1 = h.alpha_g1; pk.vk.beta_g2 = h.beta_g2; pk.vk.gamma_g2 = h.gamma_g2; pk.vk.delta_g2 = h.delta_g2;
        pk.beta_g1 = h.beta_g1; pk.delta_g1 = h.delta_g1;
        pk.vk.gamma_abc_g1 = g1_section(h.n_public + 1, 3);
        pk.a_query = g1_section(h.n_vars, 5);
        pk.b_g1_query = g1_section(h.n_vars, 6);
        pk.b_g2_query = g2_section(h.n_vars, 7);
        pk.l_query = g1_section(h.n_vars - h.n_public - 1, 8);
        pk.h_query = g1_section(h.domain_size, 9);
        return pk;
    }

    ConstraintMatrices matrices() {                     // src/zkey.rs:151-196
        Header h = groth_header();
        seek(4);
        uint32_t ncoef = detail::read_le<uint32_t>(r_);
        std::vector<Matrix> m(2, Matrix(h.domain_size));
        uint32_t max_c = 0;
        const uint64_t one[4] = {1, 0, 0, 0};
        for (uint32_t i = 0; i < ncoef; i++) {
            uint32_t matrix = detail::read_le<uint32_t>(r_), constraint = detail::read_le<uint32_t>(r_), signal = detail::read_le<uint32_t>(r_);
            BigInt256 raw; detail::read_exact(r_, raw.l, 32);
            if (matrix > 1 || constraint >= h.domain_size) throw SerializationError("bad coefficient record");
            // stored = v * R^2; the reader strips one R (zkey.rs:320-325): Montgomery residue of v = stored * R^-1
            Fr v; detail::fr_mont_mul(v.l, raw.l, one);
            if (constraint > max_c) max_c = constraint;
            m[matrix][constraint].push_back({v, (size_t)signal});
        }
        if (max_c < h.n_public) throw SerializationError("malformed zkey: no constraints");
        size_t nc = max_c - h.n_public;                 // zkey.rs:171
        for (auto& mm : m) mm.resize(nc);               // public-input rows dropped, arkworks re-adds them (qap.rs:46-50)
        ConstraintMatrices cm;
        cm.num_instance_variables = h.n_public + 1; cm.num_witness_variables = h.n_vars - h.n_public - 1; cm.num_constraints = nc;
        cm.a = std::move(m[0]); cm.b = std::move(m[1]);
        for (auto& row : cm.a) cm.a_num_non_zero += row.size();
        for (auto& row : cm.b) cm.b_num_non_zero += row.size();
        return cm;
    }

    struct Header { uint32_t n_vars, n_public, domain_size; G1Affine alpha_g1, beta_g1, delta_g1; G2Affine beta_g2, gamma_g2, delta_g2; };
    Header groth_header() {                             // src/zkey.rs:282-318
        seek(2);
        Header h;
        uint32_t n8q = detail::read_le<uint32_t>(r_);
        if (n8q != 32) throw SerializationError("unsupported base field size");
        uint64_t q[4]; detail::read_exact(r_, q, 32);
        uint32_t n8r = detail::read_le<uint32_t>(r_);
        if (n8r != 32) throw SerializationError("unsupported scalar field size");
        uint64_t r[4]; detail::read_exact(r_, r, 32);
        if (memcmp(q, detail::FQ_P, 32) || memcmp(r, detail::FR_P, 32)) throw SerializationError("only BN254 zkeys are supported");
        h.n_vars = detail::read_le<uint32_t>(r_); h.n_public = detail::read_le<uint32_t>(r_); h.domain_size = detail::read_le<uint32_t>(r_);
        detail::read_exact(r_, &h.alpha_g1, 64); detail::read_exact(r_, &h.beta_g1, 64);
        detail::read_exact(r_, &h.beta_g2, 128); detail::read_exact(r_, &h.gamma_g2, 128);
        detail::read_exact(r_, &h.delta_g1, 64); detail::read_exact(r_, &h.delta_g2, 128);
        if (h.n_vars < h.n_public + 1) throw SerializationError("bad zkey header");
        return h;
    }

private:
    void seek(uint32_t id) {
        auto it = sections_.find(id);
        if (it == sections_.end()) throw SerializationError("missing zkey section " + std::to_string(id));
        r_.clear(); r_.seekg((std::streamoff)it->second[0].position);
    }
    // points are already Montgomery (zkey.rs:327-332): one bulk read per section instead of per-point byteorder calls.
    // NB the reference checks every point on-curve (G1Affine::new, zkey.rs:347); here b2g_pk_load takes them as given.
    std::vector<G1Affine> g1_section(size_t n, uint32_t id) { seek(id); std::vector<G1Affine> v(n); if (n) detail::read_exact(r_, v.data(), n * 64); return v; }
    std::vector<G2Affine> g2_section(size_t n, uint32_t id) { seek(id); std::vector<G2Affine> v(n); if (n) detail::read_exact(r_, v.data(), n * 128); return v; }

    std::istream& r_;
    std::string ftype_;
    uint32_t version_ = 0;
    std::map<uint32_t, std::vector<detail::Section>> sections_;
};

inline std::pair<ProvingKey, ConstraintMatrices> read_zkey(std::istream& reader) {   // src/zkey.rs:53-60
    BinFile f(reader);
    ProvingKey pk = f.proving_key();
    ConstraintMatrices m = f.matrices();
    return {std::move(pk), std::move(m)};
}

// snarkjs .wtns: "wtns", version, sections {1: n8 u32, prime[n8], nWitness u32; 2: nWitness x n8 canonical LE}
inline std::vector<Fr> read_wtns(std::istream& r) {
    char magic[4]; detail::read_exact(r, magic, 4);
    if (memcmp(magic, "wtns", 4)) throw SerializationError("not a wtns file");
    detail::read_le<uint32_t>(r);
    uint32_t nsec = detail::read_le<uint32_t>(r), nwit = 0;
    std::vector<Fr> out;
    for (uint32_t i = 0; i < nsec; i++) {
        uint32_t id = detail::read_le<uint32_t>(r); uint64_t len = detail::read_le<uint64_t>(r);
        std::streamoff pos = r.tellg();
        if (id == 1) {
            uint32_t n8 = detail::read_le<uint32_t>(r);
            uint64_t prime[4]; if (n8 != 32) throw SerializationError("unsupported field size"); detail::read_exact(r, prime, 32);
            if (memcmp(prime, detail::FR_P, 32)) throw SerializationError("only BN254 witnesses are supported");
            nwit = detail::read_le<uint32_t>(r);
        } else if (id == 2) {
            out.resize(nwit);
            for (uint32_t k = 0; k < nwit; k++) { BigInt256 b; detail::read_exact(r, b.l, 32); out[k] = Fr::from_bigint(b); }
        }
        r.seekg(pos + (std::streamoff)len);
    }
    return out;
}

// ---------------------------------------------------------------------------------------------- .ptau reader (host)
// The points of a powers-of-tau ceremony of size 2^power (snarkjs .ptau sections 2-6; layout restated in ptau.py), affine
// Montgomery as in a zkey.  The vectors may hold only a prefix of the ceremony: see read_ptau.
// The prepared Lagrange sections 12-15 (snarkjs powersoftau prepare phase2; layout in ptau.py and include/b2groth.h): block k
// of a section starts at point 2^k - 1 and holds iNTT_(2^k) of the first 2^k points of its monomial array.
struct LagrangePoints {
    uint32_t power = 0;                                         // the power they were prepared at (block power + 1 padded)
    std::vector<G1Affine> tau_g1, alpha_tau_g1, beta_tau_g1;    // blocks 0 .. power + 1, 0 .. power, 0 .. power in the file
    std::vector<G2Affine> tau_g2;                               // blocks 0 .. power
};

struct Powers {
    uint32_t power = 0, ceremony_power = 0;
    std::vector<G1Affine> tau_g1, alpha_tau_g1, beta_tau_g1;    // 2^(power+1) - 1, 2^power, 2^power points in the file
    std::vector<G2Affine> tau_g2;                               // 2^power
    G2Affine beta_g2;
    bool prepared = false;                                      // lagrange holds sections 12-15 (or their prefix)
    LagrangePoints lagrange;
};

// Parses a .ptau container with the checks of ptau.read_ptau (magic, version 1, BN254's field, sections 1-6 present, not
// truncated, sizes that agree with the power), throwing SerializationError.  log_n > 0: read only the prefix a circuit
// of domain 2^log_n needs (2n - 1 / n / n / n points), so a large ceremony file is not read whole; it must not exceed the
// file's power.  log_n = 0: every point.  When sections 12-15 are all present with the sizes of the power, their blocks up to
// log_n (+ 1 for tau_g1) are read too (prepared = true); below the power tau_g1 then keeps 2n points, as the top block reads.
inline Powers read_ptau(std::istream& r, uint32_t log_n = 0) {
    r.seekg(0, std::ios::end);
    const uint64_t size = (uint64_t)r.tellg();
    r.seekg(0);
    char magic[4];
    if (size < 12) throw SerializationError("ptau: bad magic (not a .ptau file)");
    detail::read_exact(r, magic, 4);
    if (memcmp(magic, "ptau", 4)) throw SerializationError("ptau: bad magic (not a .ptau file)");
    const uint32_t version = detail::read_le<uint32_t>(r), nsec = detail::read_le<uint32_t>(r);
    if (version != 1) throw SerializationError("ptau: unsupported version " + std::to_string(version) + " (expected 1)");
    std::map<uint32_t, detail::Section> secs;
    uint64_t at = 12;
    for (uint32_t k = 0; k < nsec; k++) {
        if (at + 12 > size) throw SerializationError("ptau: section header " + std::to_string(k) + " is truncated");
        r.seekg((std::streamoff)at);
        const uint32_t id = detail::read_le<uint32_t>(r);
        const uint64_t len = detail::read_le<uint64_t>(r);
        at += 12;
        if (len > size - at) throw SerializationError("ptau: section " + std::to_string(id) + " is truncated");
        secs.insert({id, {at, len}});
        at += len;
    }
    for (uint32_t id = 1; id <= 6; id++)
        if (!secs.count(id)) throw SerializationError("ptau: section " + std::to_string(id) + " is missing");
    r.seekg((std::streamoff)secs[1].position);
    const uint32_t n8 = detail::read_le<uint32_t>(r);
    if (n8 != 32) throw SerializationError("ptau: field element size " + std::to_string(n8) + " is not BN254's (32)");
    if (secs[1].size != 44) throw SerializationError("ptau: section 1 holds " + std::to_string(secs[1].size) + " bytes, not 44");
    uint64_t q[4]; detail::read_exact(r, q, 32);
    if (memcmp(q, detail::FQ_P, 32)) throw SerializationError("ptau: the curve's base field is not BN254's");
    Powers p;
    p.power = detail::read_le<uint32_t>(r);
    p.ceremony_power = detail::read_le<uint32_t>(r);
    if (p.power < 1 || p.power > 28) throw SerializationError("ptau: power " + std::to_string(p.power) + " is out of range (1..28)");
    if (log_n > p.power) throw SerializationError("ptau: the circuit's domain 2^" + std::to_string(log_n) + " exceeds the ceremony's 2^" + std::to_string(p.power));
    const uint64_t n = 1ull << p.power, m = log_n ? 1ull << log_n : n;
    const uint64_t lag_counts[4] = {4 * n - 1, 2 * n - 1, 2 * n - 1, 2 * n - 1}, lag_rows[4] = {64, 128, 64, 64};
    p.prepared = true;
    for (int k = 0; k < 4; k++) {
        auto it = secs.find(12 + k);
        p.prepared = p.prepared && it != secs.end() && it->second.size == lag_counts[k] * lag_rows[k];
    }
    const uint64_t counts[5] = {2 * n - 1, n, n, n, 1}, rows[5] = {64, 128, 64, 64, 128};
    const uint64_t reads[5] = {2 * m - 1 + (p.prepared && m < n ? 1 : 0), m, m, m, 1};
    for (int k = 0; k < 5; k++) {
        const detail::Section s = secs[2 + k];
        if (s.size != counts[k] * rows[k])
            throw SerializationError("ptau: section " + std::to_string(2 + k) + " holds " + std::to_string(s.size) + " bytes, but power " +
                                     std::to_string(p.power) + " needs " + std::to_string(counts[k] * rows[k]));
        r.seekg((std::streamoff)s.position);
        void* dst;
        switch (k) {
            case 0: p.tau_g1.resize(reads[k]); dst = p.tau_g1.data(); break;
            case 1: p.tau_g2.resize(reads[k]); dst = p.tau_g2.data(); break;
            case 2: p.alpha_tau_g1.resize(reads[k]); dst = p.alpha_tau_g1.data(); break;
            case 3: p.beta_tau_g1.resize(reads[k]); dst = p.beta_tau_g1.data(); break;
            default: dst = &p.beta_g2; break;
        }
        detail::read_exact(r, dst, reads[k] * rows[k]);
    }
    if (p.prepared) {
        p.lagrange.power = p.power;
        const uint64_t lag_reads[4] = {4 * m - 1, 2 * m - 1, 2 * m - 1, 2 * m - 1};
        p.lagrange.tau_g1.resize(lag_reads[0]); p.lagrange.tau_g2.resize(lag_reads[1]);
        p.lagrange.alpha_tau_g1.resize(lag_reads[2]); p.lagrange.beta_tau_g1.resize(lag_reads[3]);
        void* dsts[4] = {p.lagrange.tau_g1.data(), p.lagrange.tau_g2.data(), p.lagrange.alpha_tau_g1.data(), p.lagrange.beta_tau_g1.data()};
        for (int k = 0; k < 4; k++) {
            r.seekg((std::streamoff)secs[12 + k].position);
            detail::read_exact(r, dsts[k], lag_reads[k] * lag_rows[k]);
        }
    }
    return p;
}

// `snarkjs powersoftau new`: the ceremony of power p before any contribution (tau = alpha = beta = 1: every point the standard
// generator); ceremony_power 0 means p.
inline Powers new_powers_of_tau(uint32_t power, uint32_t ceremony_power = 0) {
    if (power < 1 || power > 28) throw std::invalid_argument("new_powers_of_tau: power " + std::to_string(power) + " is outside 1..28");
    static const uint64_t G1[8] = {0xd35d438dc58f0d9dULL, 0x0a78eb28f5c70b3dULL, 0x666ea36f7879462cULL, 0x0e0a77c19a07df2fULL,
                                   0xa6ba871b8b1e1b3aULL, 0x14f1d651eb8e167bULL, 0xccdd46def0f28c58ULL, 0x1c14ef83340fbe5eULL};
    static const uint64_t G2[16] = {0x8e83b5d102bc2026ULL, 0xdceb1935497b0172ULL, 0xfbb8264797811adfULL, 0x19573841af96503bULL,
                                    0xafb4737da84c6140ULL, 0x6043dd5a5802d8c4ULL, 0x09e950fc52a02f86ULL, 0x14fef0833aea7b6bULL,
                                    0x619dfa9d886be9f6ULL, 0xfe7fd297f59e9b78ULL, 0xff9e1a62231b7dfeULL, 0x28fd7eebae9e4206ULL,
                                    0x64095b56c71856eeULL, 0xdc57f922327d3cbbULL, 0x55f935be33351076ULL, 0x0da4a0e693fd6482ULL};
    G1Affine g1; G2Affine g2;
    memcpy(&g1, G1, 64); memcpy(&g2, G2, 128);
    const size_t n = (size_t)1 << power;
    Powers p;
    p.power = power; p.ceremony_power = ceremony_power ? ceremony_power : power;
    p.tau_g1.assign(2 * n - 1, g1); p.tau_g2.assign(n, g2); p.alpha_tau_g1.assign(n, g1); p.beta_tau_g1.assign(n, g1);
    p.beta_g2 = g2;
    return p;
}

// Writes `p` as a .ptau container (sections 1-6, and 12-15 when prepared), as ptau.write_ptau does: the vectors must hold the
// full counts of p.power (a prefix is refused with std::invalid_argument).  Section 7, the contribution transcript, is not
// written.
inline void write_ptau(std::ostream& w, const Powers& p) {
    const uint64_t n = 1ull << p.power;
    if (p.power < 1 || p.power > 28 || p.tau_g1.size() != 2 * n - 1 || p.tau_g2.size() != n || p.alpha_tau_g1.size() != n ||
        p.beta_tau_g1.size() != n)
        throw std::invalid_argument("write_ptau: the arrays do not hold the counts of power " + std::to_string(p.power));
    if (p.prepared && (p.lagrange.power != p.power || p.lagrange.tau_g1.size() != 4 * n - 1 || p.lagrange.tau_g2.size() != 2 * n - 1 ||
                       p.lagrange.alpha_tau_g1.size() != 2 * n - 1 || p.lagrange.beta_tau_g1.size() != 2 * n - 1))
        throw std::invalid_argument("write_ptau: the Lagrange sections do not hold the counts of power " + std::to_string(p.power));
    auto put32 = [&](uint32_t v) { w.write((const char*)&v, 4); };
    auto put64 = [&](uint64_t v) { w.write((const char*)&v, 8); };
    auto section = [&](uint32_t id, const void* data, uint64_t bytes) { put32(id); put64(bytes); w.write((const char*)data, (std::streamsize)bytes); };
    w.write("ptau", 4);
    put32(1);
    put32(p.prepared ? 10 : 6);
    put32(1); put64(44); put32(32);
    w.write((const char*)detail::FQ_P, 32);
    put32(p.power); put32(p.ceremony_power);
    section(2, p.tau_g1.data(), p.tau_g1.size() * 64);
    section(3, p.tau_g2.data(), p.tau_g2.size() * 128);
    section(4, p.alpha_tau_g1.data(), p.alpha_tau_g1.size() * 64);
    section(5, p.beta_tau_g1.data(), p.beta_tau_g1.size() * 64);
    section(6, &p.beta_g2, 128);
    if (p.prepared) {
        section(12, p.lagrange.tau_g1.data(), p.lagrange.tau_g1.size() * 64);
        section(13, p.lagrange.tau_g2.data(), p.lagrange.tau_g2.size() * 128);
        section(14, p.lagrange.alpha_tau_g1.data(), p.lagrange.alpha_tau_g1.size() * 64);
        section(15, p.lagrange.beta_tau_g1.data(), p.lagrange.beta_tau_g1.size() * 64);
    }
    if (!w) throw SerializationError("write_ptau: the write failed");
}

// ---------------------------------------------------------------------------------------------- device side
// One Gpu = one b2g_ctx (one in-flight proof on one device).  Keys / matrices are uploaded on first use; the handle lives
// in the host object's DeviceSlot (freed with it), never in an address-keyed table.  A Gpu must outlive the proofs issued
// on it, not the keys: b2g_pk_free / b2g_matrices_free need only the device.
class Gpu {
public:
    explicit Gpu(int device = 0) { check(b2g_ctx_create(device, 0, 1, &ctx_)); }
    ~Gpu() { if (ctx_) b2g_ctx_destroy(ctx_); }
    Gpu(const Gpu&) = delete; Gpu& operator=(const Gpu&) = delete;
    static Gpu& instance() { static Gpu g(0); return g; }
    static Gpu& on(int device) {                                       // one shared context per device (device 0: instance())
        if (device == 0) return instance();
        static std::map<int, std::unique_ptr<Gpu>> gpus;
        auto& g = gpus[device];
        if (!g) g.reset(new Gpu(device));
        return *g;
    }
    b2g_ctx* ctx() { return ctx_; }

    // the b2g_pk_desc of a key (pointing into it)
    static b2g_pk_desc pk_desc(const ProvingKey& k) {
        b2g_pk_desc d; memset(&d, 0, sizeof d);
        d.n_vars = (uint32_t)k.a_query.size(); d.n_public = (uint32_t)k.vk.gamma_abc_g1.size() - 1; d.domain_size = (uint32_t)k.h_query.size();
        d.alpha_g1 = &k.vk.alpha_g1; d.beta_g1 = &k.beta_g1; d.delta_g1 = &k.delta_g1; d.beta_g2 = &k.vk.beta_g2; d.delta_g2 = &k.vk.delta_g2;
        d.a_query = k.a_query.data(); d.b_g1_query = k.b_g1_query.data(); d.b_g2_query = k.b_g2_query.data();
        d.l_query = k.l_query.data(); d.h_query = k.h_query.data();
        return d;
    }

    b2g_pk* pk(const ProvingKey& k) {
        if (void* h = k.device.find(ctx_, 0)) return (b2g_pk*)h;
        const b2g_pk_desc d = pk_desc(k);
        b2g_pk* h = nullptr; check(b2g_pk_load(ctx_, &d, &h));
        k.device.put(ctx_, 0, h, [](void* p) { b2g_pk_free((b2g_pk*)p); });
        return h;
    }

    b2g_mat* mat(const ConstraintMatrices& m, size_t n_vars, uint32_t reduction = B2G_REDUCTION_CIRCOM) {
        const uint32_t tag = reduction | (uint32_t)(n_vars << 1);     // a matrices handle is specific to (reduction, n_vars)
        if (void* h = m.device.find(ctx_, tag)) return (b2g_mat*)h;
        const MatDesc md(m, n_vars, reduction);
        b2g_mat* h = nullptr; check(b2g_matrices_load(ctx_, &md.d, &h));
        m.device.put(ctx_, tag, h, [](void* p) { b2g_matrices_free((b2g_mat*)p); });
        return h;
    }

    // the b2g_mat_desc of matrices and the CSR arrays it points into; with_c: C whatever the reduction (b2g_setup reads it for both)
    struct MatDesc {
        std::vector<uint32_t> rp[3], col[3]; std::vector<Fr> val[3];
        b2g_mat_desc d;
        MatDesc(const ConstraintMatrices& m, size_t n_vars, uint32_t reduction, bool with_c = false) {
            const Matrix* src[3] = {&m.a, &m.b, &m.c};
            const int nmat = with_c || reduction == B2G_REDUCTION_LIBSNARK ? 3 : 2;
            for (int k = 0; k < nmat; k++) {
                rp[k].assign(m.num_constraints + 1, 0);
                for (size_t i = 0; i < m.num_constraints; i++) {
                    const auto& row = i < src[k]->size() ? (*src[k])[i] : Matrix::value_type();
                    for (const auto& e : row) { val[k].push_back(e.first); col[k].push_back((uint32_t)e.second); }
                    rp[k][i + 1] = (uint32_t)col[k].size();
                }
            }
            memset(&d, 0, sizeof d);
            d.num_constraints = (uint32_t)m.num_constraints; d.num_inputs = (uint32_t)m.num_instance_variables; d.n_vars = (uint32_t)n_vars;
            d.reduction = reduction;
            d.a_rowptr = rp[0].data(); d.a_col = col[0].data(); d.a_val = val[0].data();
            d.b_rowptr = rp[1].data(); d.b_col = col[1].data(); d.b_val = val[1].data();
            if (nmat == 3) { d.c_rowptr = rp[2].data(); d.c_col = col[2].data(); d.c_val = val[2].data(); }
        }
        MatDesc(const MatDesc&) = delete;
        MatDesc& operator=(const MatDesc&) = delete;
    };

private:
    b2g_ctx* ctx_ = nullptr;
};

template <uint32_t REDUCTION>
struct Reduction {
    static constexpr uint32_t ID = REDUCTION;
    static std::vector<Fr> witness_map_from_matrices(const ConstraintMatrices& matrices, size_t num_inputs, size_t num_constraints,
                                                     const std::vector<Fr>& full_assignment, Gpu& gpu = Gpu::instance()) {
        if (num_inputs != matrices.num_instance_variables || num_constraints != matrices.num_constraints)
            throw SynthesisError("num_inputs / num_constraints disagree with the matrices");
        size_t n = 1; while (n < num_constraints + num_inputs) n <<= 1;
        if (n > (size_t(1) << 27)) throw PolynomialDegreeTooLarge();
        std::vector<Fr> h(n);
        uint32_t dom = 0;
        check(b2g_witness_map(gpu.ctx(), gpu.mat(matrices, full_assignment.size(), REDUCTION), full_assignment.data(), h.data(), &dom));
        return h;
    }
};
typedef Reduction<B2G_REDUCTION_CIRCOM> CircomReduction;       // src/circom/qap.rs:12-14 (snarkjs keys)
typedef Reduction<B2G_REDUCTION_LIBSNARK> LibsnarkReduction;   // ark-groth16's default QAP (tests/groth16.rs:9,25-35; needs matrices.c)

// ---------------------------------------------------------------------------------------------- circom 2 witnesses
// WitnessCalculator (src/witness/witness_calculator.rs) with the circuit's .wasm run by the library's device interpreter
// (b2g_wasm_load / b2g_witness_calculate): one lane per witness, many witnesses per call.  Input values are reduced
// mod r; names are hashed with FNV-1a 64.  A lane that calls the circuit's exceptionHandler stops there.
struct WitnessError : std::runtime_error {
    uint32_t status;
    WitnessError(uint32_t st, const std::string& m) : std::runtime_error(m), status(st) {}
};

class WitnessCalculator {
public:
    typedef std::vector<std::pair<std::string, std::vector<BigInt256>>> Inputs;   // (name, values), in order
    uint32_t n32 = 0, n64 = 4, witness_size = 0, input_size = 0, version = 0;

    explicit WitnessCalculator(const std::vector<uint8_t>& wasm, Gpu& gpu = Gpu::instance()) : gpu_(gpu) {
        check(b2g_wasm_load(gpu.ctx(), wasm.data(), wasm.size(), &h_));
        b2g_wasm_summary s; check(b2g_wasm_info(h_, &s));
        n32 = s.n32; witness_size = s.witness_size; input_size = s.input_size; version = s.version;
    }
    static WitnessCalculator from_file(const std::string& path, Gpu& gpu = Gpu::instance()) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw SerializationError("cannot open " + path);
        return WitnessCalculator(std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>()), gpu);
    }
    ~WitnessCalculator() { if (h_) b2g_wasm_free(h_); }
    WitnessCalculator(WitnessCalculator&& o) noexcept : n32(o.n32), n64(o.n64), witness_size(o.witness_size), input_size(o.input_size),
        version(o.version), gpu_(o.gpu_), h_(o.h_) { o.h_ = nullptr; }
    WitnessCalculator(const WitnessCalculator&) = delete;
    WitnessCalculator& operator=(const WitnessCalculator&) = delete;
    b2g_wasm* handle() const { return h_; }

    static uint64_t fnv(const std::string& name) {
        uint64_t h = 0xcbf29ce484222325ULL;
        for (unsigned char c : name) { h ^= c; h *= 0x100000001b3ULL; }
        return h;
    }
    static const char* status_name(uint32_t st) {
        static const char* const ex[7] = {"Unknown error", "Signal not found", "Too many signals set", "Signal already set",
                                          "Assert Failed", "Not enough memory", "Input signal array access exceeds the size"};
        static const char* const tr[9] = {"ok", "unreachable executed", "memory access out of bounds", "integer divide by zero",
                                          "integer overflow", "call stack exhausted", "instruction budget (fuel) exhausted",
                                          "bad call_indirect", "getWitnessSize disagrees with the module's witness size"};
        if (st >= B2G_WASM_EXCEPTION) return ex[st - B2G_WASM_EXCEPTION < 7 ? st - B2G_WASM_EXCEPTION : 0];
        return st < 9 ? tr[st] : "unknown status";
    }

    // many witnesses with the same input names and lengths: out[i] (Montgomery Fr, witness_size each) and status[i]
    void calculate_witnesses(const std::vector<Inputs>& batch, std::vector<std::vector<Fr>>& out, std::vector<uint32_t>& status,
                             bool sanity_check = false) {
        const size_t count = batch.size();
        out.assign(count, std::vector<Fr>());
        status.assign(count, 0);
        if (!count) return;
        std::vector<uint64_t> hashes; std::vector<uint32_t> counts;
        for (const auto& in : batch[0]) { hashes.push_back(fnv(in.first)); counts.push_back((uint32_t)in.second.size()); }
        std::vector<BigInt256> vals;
        for (size_t i = 0; i < count; i++) {
            if (batch[i].size() != hashes.size()) throw std::invalid_argument("calculate_witnesses: inputs differ in shape");
            for (size_t k = 0; k < batch[i].size(); k++) {
                if (fnv(batch[i][k].first) != hashes[k] || batch[i][k].second.size() != counts[k])
                    throw std::invalid_argument("calculate_witnesses: inputs differ in shape");
                for (BigInt256 v : batch[i][k].second) {
                    while (detail::geq(v.l, detail::FR_P)) {            // v mod r (v < 2^256 < 6 r)
                        unsigned __int128 br = 0;
                        for (int j = 0; j < 4; j++) {
                            const unsigned __int128 t = (unsigned __int128)v.l[j] - detail::FR_P[j] - br;
                            v.l[j] = (uint64_t)t; br = (t >> 64) & 1;
                        }
                    }
                    vals.push_back(v);
                }
            }
        }
        std::vector<Fr> flat((size_t)count * witness_size);
        check(b2g_witness_calculate(gpu_.ctx(), h_, (uint32_t)count, (uint32_t)hashes.size(), hashes.data(), counts.data(),
                                    vals.empty() ? nullptr : vals.data(), sanity_check ? 1 : 0, flat.data(), status.data()));
        for (size_t i = 0; i < count; i++) out[i].assign(flat.begin() + i * witness_size, flat.begin() + (i + 1) * witness_size);
    }
    // calculate_witness_element: one witness as field elements; throws WitnessError naming the exception or trap
    std::vector<Fr> calculate_witness_element(const Inputs& inputs, bool sanity_check = false) {
        std::vector<std::vector<Fr>> out; std::vector<uint32_t> st;
        calculate_witnesses({inputs}, out, st, sanity_check);
        if (st[0]) throw WitnessError(st[0], status_name(st[0]));
        return out[0];
    }

private:
    Gpu& gpu_;
    b2g_wasm* h_ = nullptr;
};

}  // namespace ark_circom
#include "ark_circom_verifier.hpp"
#include "ark_circom_ethereum.hpp"
namespace ark_circom {

// the b2g_vk_desc of a prepared key (pointing into pvk.vk)
inline b2g_vk_desc vk_desc(const PreparedVerifyingKey& pvk) {
    b2g_vk_desc d; memset(&d, 0, sizeof d);
    d.n_public = (uint32_t)(pvk.vk.gamma_abc_g1.size() - 1);
    d.alpha_g1 = &pvk.vk.alpha_g1; d.beta_g2 = &pvk.vk.beta_g2; d.gamma_g2 = &pvk.vk.gamma_g2; d.delta_g2 = &pvk.vk.delta_g2;
    d.gamma_abc_g1 = pvk.vk.gamma_abc_g1.data();
    return d;
}

// the key prepared on the device at first use (b2g_vk_load), kept in pvk.device
inline b2g_vk* device_vk(const PreparedVerifyingKey& pvk, Gpu& gpu) {
    if (void* h = pvk.device.find(gpu.ctx(), 0)) return (b2g_vk*)h;
    const b2g_vk_desc d = vk_desc(pvk);
    b2g_vk* vk = nullptr;
    check(b2g_vk_load(gpu.ctx(), &d, &vk));
    pvk.device.put(gpu.ctx(), 0, vk, [](void* p) { b2g_vk_free((b2g_vk*)p); });
    return vk;
}

// the keys of pvks not yet on gpu's device, prepared in ONE b2g_vk_load_many call and kept in each pvk.device as device_vk
// keeps them (a key given twice loads once).  When the library refuses a key, nothing is loaded and a DeviceError carries
// the message b2g_vk_load gives for that key alone, after "key i: " (i = its first index in pvks) when name_key is set.
inline void device_vks(const std::vector<const PreparedVerifyingKey*>& pvks, Gpu& gpu, bool name_key) {
    std::vector<const PreparedVerifyingKey*> todo;
    std::vector<size_t> at;
    std::vector<b2g_vk_desc> descs;
    for (size_t i = 0; i < pvks.size(); i++) {
        const PreparedVerifyingKey* p = pvks[i];
        if (p->device.find(gpu.ctx(), 0) || std::find(todo.begin(), todo.end(), p) != todo.end()) continue;
        todo.push_back(p); at.push_back(i); descs.push_back(vk_desc(*p));
    }
    if (todo.empty()) return;
    std::vector<b2g_vk*> vks(todo.size());
    const int rc = b2g_vk_load_many(gpu.ctx(), (uint32_t)todo.size(), descs.data(), vks.data());
    if (rc != B2G_OK) {
        // "b2g_vk_load_many: key k: <b2g_vk_load's message>" names the key; other messages name none
        std::string msg = b2g_last_error();
        const std::string head = "b2g_vk_load_many: key ";
        size_t k = 0;
        if (msg.compare(0, head.size(), head) == 0) {
            size_t len = 0;
            k = std::stoul(msg.substr(head.size()), &len);
            msg = msg.substr(head.size() + len + 2);
            if (name_key) msg = "key " + std::to_string(at[k]) + ": " + msg;
        }
        throw DeviceError(std::string("b2groth error ") + std::to_string(rc) + ": " + msg);
    }
    for (size_t i = 0; i < todo.size(); i++) todo[i]->device.put(gpu.ctx(), 0, vks[i], [](void* p) { b2g_vk_free((b2g_vk*)p); });
}

// what the Groth16 verifiers share: the argument checks, the key on the device (device_vk; left to the caller unless
// `load`) and the encoded public inputs and proofs (P = Proof, 256-byte rows, or CompressedProof, 128-byte rows)
struct VerifyCall {
    size_t n = 0;
    Gpu* gpu = nullptr;
    b2g_vk* vk = nullptr;
    std::vector<BigInt256> pub;
    std::vector<uint8_t> bytes;
    template <class P>
    VerifyCall(const char* fn, const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
               const std::vector<P>& proofs, int device, bool load = true) {
        static_assert(sizeof(P) == 256 || sizeof(P) == 128, "a proof row is 256 bytes, or 128 compressed");
        if (public_inputs.size() != proofs.size()) throw SynthesisError(std::string(fn) + ": one public-input list per proof");
        const size_t n_public = pvk.vk.gamma_abc_g1.size() - 1;
        if (proofs.empty()) return;
        for (const auto& xs : public_inputs) if (xs.size() != n_public) throw MalformedVerifyingKey();
        n = proofs.size();
        gpu = &Gpu::on(device);
        if (load) vk = device_vk(pvk, *gpu);
        pub.resize(n * n_public);
        for (size_t i = 0; i < n; i++) for (size_t k = 0; k < n_public; k++) pub[i * n_public + k] = public_inputs[i][k].into_bigint();
        bytes.resize(n * sizeof(P));
        for (size_t i = 0; i < n; i++) memcpy(&bytes[i * sizeof(P)], &proofs[i], sizeof(P));
    }
};

// The verdict of Groth16T::verify_powers_of_tau (b2g_powers_check): ok, or the reason of the failure in the messages of
// b2g_setup_from_powers ("tau_g2[17]: not in G2"), or "the powers are not those of one tau, alpha and beta".
struct PowersCheck {
    bool ok = false;
    int rule = 0;                 // b2g_powers_report's rule code
    std::string array;            // rules 1-5: the array and the index of the first failing point; rule 7: the section
    uint64_t index = 0;
    explicit operator bool() const { return ok; }
    std::string reason() const {
        if (ok) return "";
        if (rule == 6) return "the powers are not those of one tau, alpha and beta";
        if (rule == 7) return array + " is not the transform of " + array.substr(9);
        const bool g2 = array == "tau_g2" || array == "beta_g2" || array == "lagrange_tau_g2";
        static const char* const texts[6] = {"", "a coordinate >= p", "off the curve", "at infinity", "not in G2", "not the generator"};
        return array + "[" + std::to_string(index) + "]: " + (rule == 2 && g2 ? "off the twist" : texts[rule]);
    }
};

// The verdict of Groth16T::verify_proving_key (b2g_setup_check): ok, or the reason of the failure in the words of
// keycheck.py ("l_query[17]: off the curve", "alpha_g1 is not the ceremony's", "b_g2_query does not match the circuit and
// ceremony", "matrix A differs from the circuit at row 17").
struct SetupCheck {
    bool ok = false;
    std::string why;
    explicit operator bool() const { return ok; }
    const std::string& reason() const { return why; }
};

namespace detail {
// the rows of a matrix sorted by column, duplicates summed mod r, zeros dropped (Montgomery values compare as canonical ones)
inline std::vector<std::vector<std::pair<size_t, Fr>>> canonical_rows(const Matrix& m, size_t rows) {
    std::vector<std::vector<std::pair<size_t, Fr>>> out(rows);
    for (size_t r = 0; r < rows && r < m.size(); r++) {
        std::map<size_t, Fr> acc;
        for (const auto& e : m[r]) {
            Fr& a = acc[e.second];
            u128 c = 0;
            uint64_t t[4];
            for (int i = 0; i < 4; i++) { c += (u128)a.l[i] + e.first.l[i]; t[i] = (uint64_t)c; c >>= 64; }
            if (c || geq(t, FR_P)) { u128 br = 0; for (int i = 0; i < 4; i++) { u128 d = (u128)t[i] - FR_P[i] - (uint64_t)br; t[i] = (uint64_t)d; br = (d >> 64) & 1; } }
            memcpy(a.l, t, 32);
        }
        for (const auto& kv : acc) if (!kv.second.is_zero()) out[r].push_back(kv);
    }
    return out;
}
}  // namespace detail

// the five challenges of the ceremony check (rho, sigma, pi, kappa, eps), uniform in [1, r), from std::random_device
inline std::vector<BigInt256> powers_challenges(size_t count = 5) {
    std::random_device rd;
    std::vector<BigInt256> c(count);
    for (BigInt256& b : c) {
        do {
            for (int t = 0; t < 4; t++) b.l[t] = ((uint64_t)rd() << 32) | rd();
            b.l[3] &= 0x3FFFFFFFFFFFFFFFULL;
        } while (detail::geq(b.l, detail::FR_P) || !(b.l[0] | b.l[1] | b.l[2] | b.l[3]));
    }
    return c;
}

// n nonzero 128-bit weights of the batch check (4 little-endian words each) from std::random_device
inline std::vector<uint32_t> batch_weights(size_t n) {
    std::random_device rd;
    std::vector<uint32_t> w(4 * n);
    for (size_t i = 0; i < n; i++) {
        do { for (int t = 0; t < 4; t++) w[4 * i + t] = (uint32_t)rd(); } while (!(w[4 * i] | w[4 * i + 1] | w[4 * i + 2] | w[4 * i + 3]));
    }
    return w;
}

// one batch of Groth16::verify_batch_keys: a prepared key with its proofs (P = Proof, or CompressedProof) and their public
// inputs; the same key may appear in several batches
template <class P>
struct KeyBatchOf {
    const PreparedVerifyingKey& pvk;
    const std::vector<std::vector<Fr>>& public_inputs;
    const std::vector<P>& proofs;
};
typedef KeyBatchOf<Proof> KeyBatch;
typedef KeyBatchOf<CompressedProof> CompressedKeyBatch;

// the b2g_key_batch rows of the keyed verifiers for the batches that hold proofs (row i is batch at[i]), with the arrays
// they point into; weights from std::random_device.  Every batch's checks run first, in batch order, up to the first batch
// that fails them; the keys of the batches before it that hold proofs then load in ONE b2g_vk_load_many call (device_vks).
// A refused key throws; otherwise the failing batch throws its own error: the errors, and which of them wins, are those of
// loading each batch's key as the batch is reached.
struct KeysTable {
    std::vector<VerifyCall> calls;
    std::vector<std::vector<uint32_t>> weights;
    std::vector<b2g_key_batch> table;
    std::vector<size_t> at;
    size_t total = 0;
    template <class P>
    KeysTable(const char* fn, const std::vector<KeyBatchOf<P>>& batches, int device) {
        calls.reserve(batches.size());
        std::exception_ptr failure;
        std::vector<const PreparedVerifyingKey*> pvks;
        for (size_t k = 0; k < batches.size() && !failure; k++) {
            const std::string where = std::string(fn) + ": key " + std::to_string(k);
            try {
                calls.emplace_back(where.c_str(), batches[k].pvk, batches[k].public_inputs, batches[k].proofs, device, false);
                if (calls.back().n) pvks.push_back(&batches[k].pvk);
            } catch (...) {
                failure = std::current_exception();
            }
        }
        if (!pvks.empty()) device_vks(pvks, Gpu::on(device), false);
        if (failure) std::rethrow_exception(failure);
        for (size_t k = 0; k < batches.size(); k++) {
            VerifyCall& c = calls[k];
            if (c.n == 0) continue;
            c.vk = device_vk(batches[k].pvk, *c.gpu);     // loaded above
            weights.push_back(batch_weights(c.n));
            b2g_key_batch b; memset(&b, 0, sizeof b);
            b.vk = c.vk; b.count = (uint32_t)c.n;
            b.public_inputs = c.pub.empty() ? nullptr : c.pub.data();
            b.proofs = c.bytes.data(); b.weights = weights.back().data();
            table.push_back(b);
            at.push_back(k);
            total += c.n;
        }
    }
};

// the one-key verifiers' kinds
enum class VerifyKind { many, batch, locate };

// verify_many, verify_batch, verify_batch_locate and their compressed forms (P = Proof, or CompressedProof): one ABI call,
// with weights from std::random_device when the kind takes them; the verdicts (one for batch, else one per proof), none
// for an empty batch
template <class P>
inline std::vector<bool> verify_one_key(const char* fn, VerifyKind kind, const PreparedVerifyingKey& pvk,
                                        const std::vector<std::vector<Fr>>& public_inputs, const std::vector<P>& proofs, int device) {
    VerifyCall c(fn, pvk, public_inputs, proofs, device);
    if (c.n == 0) return {};
    std::vector<uint8_t> verdicts(kind == VerifyKind::batch ? 1 : c.n);
    b2g_ctx* ctx = c.gpu->ctx();
    const void* pub = c.pub.empty() ? nullptr : c.pub.data();
    const bool z = sizeof(P) == 128;
    if (kind == VerifyKind::many) {
        check((z ? b2g_verify_many_compressed : b2g_verify_many)(ctx, c.vk, (uint32_t)c.n, pub, c.bytes.data(), verdicts.data()));
    } else {
        const std::vector<uint32_t> w = batch_weights(c.n);
        auto entry = kind == VerifyKind::batch ? (z ? b2g_verify_batch_compressed : b2g_verify_batch)
                                               : (z ? b2g_verify_batch_locate_compressed : b2g_verify_batch_locate);
        check(entry(ctx, c.vk, (uint32_t)c.n, pub, c.bytes.data(), w.data(), verdicts.data()));
    }
    return std::vector<bool>(verdicts.begin(), verdicts.end());
}

// verify_batch_keys, verify_batch_keys_locate and their compressed forms: one ABI call over the batches that hold proofs;
// per batch its verdicts (one per proof when locate, else one), none for an empty batch
template <class P>
inline std::vector<std::vector<bool>> verify_keys_call(const char* fn, const std::vector<KeyBatchOf<P>>& batches, bool locate, int device) {
    const KeysTable t(fn, batches, device);
    std::vector<std::vector<bool>> out(batches.size());
    if (t.table.empty()) return out;
    std::vector<uint8_t> verdicts(locate ? t.total : t.table.size());
    b2g_ctx* ctx = Gpu::on(device).ctx();
    const bool z = sizeof(P) == 128;
    auto entry = locate ? (z ? b2g_verify_batch_keys_locate_compressed : b2g_verify_batch_keys_locate)
                        : (z ? b2g_verify_batch_keys_compressed : b2g_verify_batch_keys);
    check(entry(ctx, (uint32_t)t.table.size(), t.table.data(), verdicts.data()));
    for (size_t i = 0, v = 0; i < t.at.size(); i++) {
        const size_t m = locate ? t.table[i].count : 1;
        out[t.at[i]].assign(verdicts.begin() + v, verdicts.begin() + v + m);
        v += m;
    }
    return out;
}

// one verdict per batch from verify_keys_call's lists: an empty batch is true
inline std::vector<bool> batch_verdicts(const std::vector<std::vector<bool>>& lists) {
    std::vector<bool> out;
    for (const auto& l : lists) out.push_back(l.empty() || l[0]);
    return out;
}

// the b2g_delta_key of a key's delta, L and H fields (the ABI reads `before` only; the pointers are not const there)
inline b2g_delta_key delta_key(const ProvingKey& pk) {
    b2g_delta_key d;
    d.n_l = (uint32_t)pk.l_query.size(); d.n_h = (uint32_t)pk.h_query.size();
    d.delta_g1 = const_cast<G1Affine*>(&pk.delta_g1); d.delta_g2 = const_cast<G2Affine*>(&pk.vk.delta_g2);
    d.l_query = pk.l_query.empty() ? nullptr : const_cast<G1Affine*>(pk.l_query.data());
    d.h_query = pk.h_query.empty() ? nullptr : const_cast<G1Affine*>(pk.h_query.data());
    return d;
}

// Proving keys loaded on one device for proving under all of them in one pass (Groth16T::load_proving_keys,
// b2g_pk_group_load).  Owns the group's device state; the keys' matrices must outlive it.
class ProvingKeyGroup {
public:
    ProvingKeyGroup(b2g_pk_group* h, std::vector<size_t> n_vars) : h_(h), n_vars_(std::move(n_vars)) {}
    ~ProvingKeyGroup() { if (h_) b2g_pk_group_free(h_); }
    ProvingKeyGroup(const ProvingKeyGroup&) = delete; ProvingKeyGroup& operator=(const ProvingKeyGroup&) = delete;
    b2g_pk_group* handle() const { return h_; }
    size_t n_keys() const { return n_vars_.size(); }
    size_t n_vars(size_t k) const { return n_vars_[k]; }
private:
    b2g_pk_group* h_;
    std::vector<size_t> n_vars_;
};

template <class QAP = CircomReduction>
struct Groth16T {                                       // Groth16::<Bn254, QAP>
    // verification (host pairing, ark_circom_verifier.hpp): src/zkey.rs:868-870, 914-916; tests/groth16.rs:33-35
    static PreparedVerifyingKey process_vk(const VerifyingKey& vk) { return prepare_verifying_key(vk); }
    static bool verify_with_processed_vk(const PreparedVerifyingKey& pvk, const std::vector<Fr>& public_inputs, const Proof& proof) {
        return ark_circom::verify_with_processed_vk(pvk, public_inputs, proof);
    }
    static bool verify(const VerifyingKey& vk, const std::vector<Fr>& public_inputs, const Proof& proof) {
        return ark_circom::verify_with_processed_vk(prepare_verifying_key(vk), public_inputs, proof);
    }
    // verify_with_processed_vk for many proofs of one key in ONE device pass (b2g_verify_many).  The key is prepared on the
    // device at first use (b2g_vk_load) and kept in pvk.device.  Verdicts equal the host call's, except for a proof
    // coordinate >= p: the host call throws SerializationError there, the batch reports the proof invalid.
    static std::vector<bool> verify_many(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                                         const std::vector<Proof>& proofs, int device = 0) {
        return verify_one_key("verify_many", VerifyKind::many, pvk, public_inputs, proofs, device);
    }
    // whether ALL proofs are valid, from one random-linear-combination pairing check (b2g_verify_batch): true iff every
    // proof passes verify_many and every B lies in G2, except with probability <= 1 / (2^128 - 1).  The 128-bit weights
    // come from std::random_device, drawn after the proofs are fixed.  On false, call verify_batch_locate to find the invalid
    // proofs.  An empty batch is true.
    static bool verify_batch(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                             const std::vector<Proof>& proofs, int device = 0) {
        const std::vector<bool> v = verify_one_key("verify_batch", VerifyKind::batch, pvk, public_inputs, proofs, device);
        return v.empty() || v[0];
    }
    // one verdict per proof at about verify_batch's cost when few proofs are invalid (b2g_verify_batch_locate): the batch
    // check runs once per group of 64 proofs over the group's well-formed proofs, and the well-formed proofs of a failing
    // group are checked as verify_many checks them.  A proof with a coordinate >= p, a point off its curve or a B outside
    // G2 is false.  A proof that verify_many accepts and whose B is in G2 is always true; any other proof is false except
    // with probability <= (groups holding such a proof) / (2^128 - 1).  Weights from std::random_device, as verify_batch.
    static std::vector<bool> verify_batch_locate(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                                                 const std::vector<Proof>& proofs, int device = 0) {
        return verify_one_key("verify_batch_locate", VerifyKind::locate, pvk, public_inputs, proofs, device);
    }
    // process_vk on the device for many keys in ONE device pass (b2g_vk_load_many), e.g. when a node starts: every key not
    // yet on the device is prepared and kept in its pvk.device, so that no verifier call has to prepare it.  A key with a point
    // off its curve throws DeviceError naming its index in pvks; then none of the keys is loaded.
    static void load_verifying_keys(const std::vector<PreparedVerifyingKey>& pvks, int device = 0) {
        std::vector<const PreparedVerifyingKey*> ptrs;
        for (const PreparedVerifyingKey& p : pvks) ptrs.push_back(&p);
        if (!ptrs.empty()) device_vks(ptrs, Gpu::on(device), true);
    }
    // verify_batch for many keys in ONE device pass (b2g_verify_batch_keys): one verdict per batch, equal to verify_batch on
    // that batch with the same weights; an invalid proof changes its own batch's verdict only, and an empty batch is true.
    // The keys not yet on the device are prepared in one b2g_vk_load_many call and kept in their pvk.device.  Weights from
    // std::random_device.
    static std::vector<bool> verify_batch_keys(const std::vector<KeyBatch>& batches, int device = 0) {
        return batch_verdicts(verify_keys_call("verify_batch_keys", batches, false, device));
    }
    // verify_batch_keys on compressed proofs, decoded on the device (b2g_verify_batch_keys_compressed): a batch with a proof
    // that does not decode is false, the others as verify_batch_keys on the decoded proofs
    static std::vector<bool> verify_batch_keys_compressed(const std::vector<CompressedKeyBatch>& batches, int device = 0) {
        return batch_verdicts(verify_keys_call("verify_batch_keys_compressed", batches, false, device));
    }
    // verify_batch_locate for many keys in ONE device pass (b2g_verify_batch_keys_locate): one verdict list per batch, equal
    // to verify_batch_locate on that batch with the same weights (groups of 64 start at each batch's first proof); an empty
    // batch gives an empty list.  Weights from std::random_device.
    static std::vector<std::vector<bool>> verify_batch_keys_locate(const std::vector<KeyBatch>& batches, int device = 0) {
        return verify_keys_call("verify_batch_keys_locate", batches, true, device);
    }
    // verify_batch_keys_locate on compressed proofs, decoded on the device (b2g_verify_batch_keys_locate_compressed): a proof
    // that does not decode is false, the others as verify_batch_keys_locate on the decoded proofs
    static std::vector<std::vector<bool>> verify_batch_keys_locate_compressed(const std::vector<CompressedKeyBatch>& batches, int device = 0) {
        return verify_keys_call("verify_batch_keys_locate_compressed", batches, true, device);
    }
    // Proof::<Bn254>::deserialize_compressed (ark-serialize 0.5, Validate::Yes) for many proofs in one device pass
    // (b2g_proofs_decompress): an empty optional where arkworks would refuse the bytes (both flag bits set, a coordinate
    // >= p, an x without a y, or a B outside G2)
    static std::vector<std::optional<Proof>> decompress_proofs(const std::vector<CompressedProof>& blobs, int device = 0) {
        if (blobs.empty()) return {};
        Gpu& gpu = Gpu::on(device);
        std::vector<Proof> rows(blobs.size());
        std::vector<uint8_t> ok(blobs.size());
        check(b2g_proofs_decompress(gpu.ctx(), (uint32_t)blobs.size(), blobs.data(), rows[0].bytes, ok.data()));
        std::vector<std::optional<Proof>> out(blobs.size());
        for (size_t i = 0; i < blobs.size(); i++) if (ok[i]) out[i] = rows[i];
        return out;
    }
    // verify_many on compressed proofs, decoded on the device (b2g_verify_many_compressed): a verdict is true exactly when
    // the proof decodes (G2 check included) and the decoded proof passes verify_many
    static std::vector<bool> verify_many_compressed(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                                                    const std::vector<CompressedProof>& blobs, int device = 0) {
        return verify_one_key("verify_many_compressed", VerifyKind::many, pvk, public_inputs, blobs, device);
    }
    // verify_batch on compressed proofs, decoded on the device (b2g_verify_batch_compressed): true exactly when every proof
    // decodes and verify_batch would be true on the decoded proofs with the same weights
    static bool verify_batch_compressed(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                                        const std::vector<CompressedProof>& blobs, int device = 0) {
        const std::vector<bool> v = verify_one_key("verify_batch_compressed", VerifyKind::batch, pvk, public_inputs, blobs, device);
        return v.empty() || v[0];
    }
    // verify_batch_locate on compressed proofs, decoded on the device (b2g_verify_batch_locate_compressed): a proof that does
    // not decode is false, the others as verify_batch_locate on the decoded proofs
    static std::vector<bool> verify_batch_locate_compressed(const PreparedVerifyingKey& pvk, const std::vector<std::vector<Fr>>& public_inputs,
                                                            const std::vector<CompressedProof>& blobs, int device = 0) {
        return verify_one_key("verify_batch_locate_compressed", VerifyKind::locate, pvk, public_inputs, blobs, device);
    }
    // Groth16::rerandomize_proof (ark-groth16 0.5.0) for many proofs of one key in ONE device pass (b2g_rerandomize_many): a
    // new proof of the same statement per proof, unlinkable to it, with no witness.  Proof i's factors are drawn from rng as
    // rerandomize_proof called on each proof in turn draws them.  An empty optional in place of a malformed proof (a
    // coordinate >= p or a point off its curve); B is not checked for membership in G2, as in arkworks.
    template <class Rng>
    static std::vector<std::optional<Proof>> rerandomize_many(const PreparedVerifyingKey& pvk, const std::vector<Proof>& proofs, Rng& rng,
                                                              int device = 0) {
        if (proofs.empty()) return {};
        Gpu& gpu = Gpu::on(device);
        const size_t n = proofs.size();
        std::vector<BigInt256> r1(n), r2(n);
        for (size_t i = 0; i < n; i++) {
            Fr a, b;
            while (a.is_zero() || b.is_zero()) { a = Fr::rand(rng); b = Fr::rand(rng); }   // r1, then r2, again while either is 0
            r1[i] = a.into_bigint(); r2[i] = b.into_bigint();
        }
        std::vector<Proof> rows(n);
        std::vector<uint8_t> ok(n);
        check(b2g_rerandomize_many(gpu.ctx(), device_vk(pvk, gpu), (uint32_t)n, proofs.data(), r1.data(), r2.data(), rows[0].bytes, ok.data()));
        std::vector<std::optional<Proof>> out(n);
        for (size_t i = 0; i < n; i++) if (ok[i]) out[i] = rows[i];
        return out;
    }
    // Groth16::rerandomize_proof(vk, proof, rng): A' = r1^-1 A, B' = r1 B + (r1 r2) delta_2, C' = C + r2 A with r1, r2 drawn
    // as arkworks draws them; throws SerializationError for a malformed proof
    template <class Rng>
    static Proof rerandomize_proof(const PreparedVerifyingKey& pvk, const Proof& proof, Rng& rng, int device = 0) {
        const std::optional<Proof> p = rerandomize_many(pvk, std::vector<Proof>{proof}, rng, device)[0];
        if (!p) throw SerializationError("rerandomize_proof: the proof is malformed (a coordinate >= p or a point off its curve)");
        return *p;
    }
    // the inputs of a prove call, one proof at a time: (r, s) as canonical integers and the witness; a witness of another
    // length than n_vars throws AssignmentMissing
    struct ProveInputs {
        std::vector<BigInt256> r, s;
        std::vector<const void*> w;
        void add(size_t n_vars, const std::pair<Fr, Fr>& rs, const std::vector<Fr>& assignment) {
            if (assignment.size() != n_vars) throw SynthesisError("AssignmentMissing: full_assignment length != n_vars");
            r.push_back(rs.first.into_bigint()); s.push_back(rs.second.into_bigint());
            w.push_back(assignment.data());
        }
    };
    static Proof create_proof_with_reduction_and_matrices(const ProvingKey& pk, const Fr& r, const Fr& s, const ConstraintMatrices& matrices,
                                                          size_t num_inputs, size_t num_constraints, const std::vector<Fr>& full_assignment,
                                                          Gpu& gpu = Gpu::instance()) {
        if (num_inputs != matrices.num_instance_variables || num_constraints != matrices.num_constraints)
            throw SynthesisError("num_inputs / num_constraints disagree with the matrices");
        ProveInputs in;
        in.add(pk.a_query.size(), {r, s}, full_assignment);
        Proof p;
        check(b2g_prove(gpu.ctx(), gpu.pk(pk), gpu.mat(matrices, full_assignment.size(), QAP::ID), in.r[0].l, in.s[0].l, full_assignment.data(), p.bytes));
        return p;
    }

    // Many proofs for one key, `inflight` of them queued on the GPU at any time, driven by THIS thread alone
    // (b2g_prove_submit / b2g_prove_wait on `inflight` contexts): what a rayon pool around the synchronous call does in the
    // reference's world.  rs[i] = (r, s) and assignments[i] = full assignment of proof i; witnesses are page-locked for the
    // duration of the call so that their upload overlaps the previous proofs.  Proofs are returned in order.
    static std::vector<Proof> prove_batch(const ProvingKey& pk, const ConstraintMatrices& matrices, const std::vector<std::pair<Fr, Fr>>& rs,
                                          const std::vector<const std::vector<Fr>*>& assignments, int inflight = 3, int device = 0) {
        if (rs.size() != assignments.size()) throw SynthesisError("prove_batch: one (r, s) per assignment");
        const size_t n = rs.size();
        if (inflight < 1) inflight = 1;
        std::vector<std::unique_ptr<Gpu>> gpus;
        for (int k = 0; k < inflight && (size_t)k < n; k++) gpus.emplace_back(new Gpu(device));
        std::vector<Proof> out(n);
        ProveInputs in;
        for (size_t i = 0; i < n; i++) {
            in.add(pk.a_query.size(), rs[i], *assignments[i]);
            check(b2g_host_register(assignments[i]->data(), assignments[i]->size() * sizeof(Fr)));
        }
        auto submit = [&](size_t i) {
            Gpu& g = *gpus[i % gpus.size()];
            check(b2g_prove_submit(g.ctx(), g.pk(pk), g.mat(matrices, assignments[i]->size(), QAP::ID), in.r[i].l, in.s[i].l, assignments[i]->data(), out[i].bytes));
        };
        size_t submitted = 0;
        try {
            for (; submitted < gpus.size(); submitted++) submit(submitted);
            for (size_t done = 0; done < n; done++) {
                check(b2g_prove_wait(gpus[done % gpus.size()]->ctx()));
                if (submitted < n) submit(submitted++);
            }
        } catch (...) {
            for (size_t i = 0; i < n; i++) b2g_host_unregister(assignments[i]->data());
            throw;
        }
        for (size_t i = 0; i < n; i++) b2g_host_unregister(assignments[i]->data());
        return out;
    }

    // Many proofs for one key in ONE device pass (b2g_prove_many): every kernel of the pipeline runs once for the whole batch.
    // Unlike prove_batch, which queues K independent proofs on K contexts, this is K proofs on one context, sorted and reduced
    // together; proofs[i] is byte-identical to create_proof_with_reduction_and_matrices(rs[i], assignments[i]).  README.md
    // gives the measured rates: it is the faster route up to 2^16 domains, prove_batch from 2^18 up.  The batch's device
    // buffers stay with `gpu`.
    static std::vector<Proof> create_proofs(const ProvingKey& pk, const ConstraintMatrices& matrices, const std::vector<std::pair<Fr, Fr>>& rs,
                                            const std::vector<const std::vector<Fr>*>& assignments, Gpu& gpu = Gpu::instance()) {
        if (rs.size() != assignments.size()) throw SynthesisError("create_proofs: one (r, s) per assignment");
        const size_t n = rs.size();
        if (n == 0) return {};
        ProveInputs in;
        for (size_t i = 0; i < n; i++) in.add(pk.a_query.size(), rs[i], *assignments[i]);
        std::vector<Proof> out(n);
        std::vector<uint8_t> bytes(n * 256);
        check(b2g_prove_many(gpu.ctx(), gpu.pk(pk), gpu.mat(matrices, pk.a_query.size(), QAP::ID), (uint32_t)n, in.r.data(), in.s.data(), in.w.data(), bytes.data()));
        for (size_t i = 0; i < n; i++) memcpy(out[i].bytes, bytes.data() + 256 * i, 256);
        return out;
    }

    // create_proofs for many keys: keys[k] = (pk, matrices) loaded with QAP's reduction into one group (b2g_pk_group_load); a
    // key may appear several times.
    static std::unique_ptr<ProvingKeyGroup> load_proving_keys(const std::vector<std::pair<const ProvingKey*, const ConstraintMatrices*>>& keys,
                                                              Gpu& gpu = Gpu::instance()) {
        std::vector<b2g_pk_desc> descs;
        std::vector<b2g_mat*> mats;
        std::vector<size_t> n_vars;
        for (const auto& k : keys) {
            descs.push_back(Gpu::pk_desc(*k.first));
            mats.push_back(gpu.mat(*k.second, k.first->a_query.size(), QAP::ID));
            n_vars.push_back(k.first->a_query.size());
        }
        b2g_pk_group* h = nullptr;
        check(b2g_pk_group_load(gpu.ctx(), (uint32_t)descs.size(), descs.data(), mats.data(), &h));
        return std::unique_ptr<ProvingKeyGroup>(new ProvingKeyGroup(h, std::move(n_vars)));
    }

    // Batches of proofs under every key of a group in ONE device pass (b2g_prove_keys): batches[k] = (rs, assignments) of key k
    // (may be empty); returns one vector of proofs per key, batch k byte-identical to create_proofs on key k.
    using KeyBatch = std::pair<std::vector<std::pair<Fr, Fr>>, std::vector<const std::vector<Fr>*>>;
    static std::vector<std::vector<Proof>> create_proofs_keys(const ProvingKeyGroup& group, const std::vector<KeyBatch>& batches,
                                                              Gpu& gpu = Gpu::instance()) {
        if (batches.size() != group.n_keys()) throw SynthesisError("create_proofs_keys: one batch per key of the group");
        std::vector<uint32_t> counts;
        ProveInputs in;
        for (size_t k = 0; k < batches.size(); k++) {
            const auto& b = batches[k];
            if (b.first.size() != b.second.size()) throw SynthesisError("create_proofs_keys: one (r, s) per assignment");
            for (size_t i = 0; i < b.first.size(); i++) in.add(group.n_vars(k), b.first[i], *b.second[i]);
            counts.push_back((uint32_t)b.first.size());
        }
        std::vector<std::vector<Proof>> out(batches.size());
        if (in.w.empty()) return out;
        std::vector<uint8_t> bytes(in.w.size() * 256);
        check(b2g_prove_keys(gpu.ctx(), group.handle(), counts.data(), in.r.data(), in.s.data(), in.w.data(), bytes.data()));
        size_t at = 0;
        for (size_t k = 0; k < batches.size(); k++) {
            out[k].resize(counts[k]);
            for (auto& p : out[k]) { memcpy(p.bytes, bytes.data() + 256 * at, 256); at++; }
        }
        return out;
    }

    // Groth16::generate_parameters_with_qap(circuit, alpha, beta, gamma, delta, g1, g2, rng) (ark-groth16 0.5) with tau given
    // instead of drawn: every scalar and point of the key on the device (b2g_setup).  g1 / g2 = nullptr: the standard
    // generators.  The matrices must carry C, as R1CS::to_matrices gives them; n_vars = num_instance + num_witness variables.
    static ProvingKey generate_parameters_with_qap(const ConstraintMatrices& matrices, const Fr& alpha, const Fr& beta, const Fr& gamma,
                                                   const Fr& delta, const G1Affine* g1, const G2Affine* g2, const Fr& tau,
                                                   Gpu& gpu = Gpu::instance()) {
        const size_t ni = matrices.num_instance_variables, nv = ni + matrices.num_witness_variables;
        if (ni == 0) throw SynthesisError("generate_parameters_with_qap: no instance variable");
        if (matrices.num_constraints && matrices.c.empty())
            throw SynthesisError("generate_parameters_with_qap needs the C matrix (R1CS route); zkey matrices have none");
        size_t n = 1;
        while (n < matrices.num_constraints + ni) n <<= 1;
        ProvingKey pk;
        pk.vk.gamma_abc_g1.resize(ni); pk.a_query.resize(nv); pk.b_g1_query.resize(nv); pk.b_g2_query.resize(nv);
        pk.l_query.resize(nv - ni); pk.h_query.resize(QAP::ID == B2G_REDUCTION_LIBSNARK ? n - 1 : n);
        BigInt256 k[5] = {alpha.into_bigint(), beta.into_bigint(), gamma.into_bigint(), delta.into_bigint(), tau.into_bigint()};
        const b2g_setup_secrets sec = {k[0].l, k[1].l, k[2].l, k[3].l, k[4].l, g1, g2};
        b2g_setup_out out = {&pk.vk.alpha_g1, &pk.beta_g1, &pk.delta_g1, &pk.vk.beta_g2, &pk.vk.gamma_g2, &pk.vk.delta_g2,
                             pk.vk.gamma_abc_g1.data(), pk.a_query.data(), pk.b_g1_query.data(), pk.b_g2_query.data(),
                             pk.l_query.data(), pk.h_query.data()};
        const Gpu::MatDesc md(matrices, nv, QAP::ID, true);
        const int rc = b2g_setup(gpu.ctx(), &md.d, &sec, &out);
        for (BigInt256& b : k) {                                // the toxic waste does not outlive the call on the host either
            volatile uint64_t* wipe = b.l;
            for (int i = 0; i < 4; i++) wipe[i] = 0;
        }
        check(rc);
        return pk;
    }
    // `snarkjs groth16 setup circuit.r1cs pot.ptau` (b2g_setup_from_powers): the key of the matrices (with C) from a ceremony,
    // gamma = delta = 1.  Throws std::invalid_argument when the powers hold fewer points than the circuit's domain reads.
    static ProvingKey generate_parameters_from_powers_of_tau(const ConstraintMatrices& matrices, const Powers& powers,
                                                             Gpu& gpu = Gpu::instance()) {
        const size_t ni = matrices.num_instance_variables, nv = ni + matrices.num_witness_variables;
        if (ni == 0) throw SynthesisError("generate_parameters_from_powers_of_tau: no instance variable");
        if (matrices.num_constraints && matrices.c.empty())
            throw SynthesisError("generate_parameters_from_powers_of_tau needs the C matrix (R1CS route); zkey matrices have none");
        size_t n = 1;
        while (n < matrices.num_constraints + ni) n <<= 1;
        if (n <= (1ull << powers.power) &&
            (powers.tau_g1.size() < 2 * n - 1 || powers.tau_g2.size() < n || powers.alpha_tau_g1.size() < n || powers.beta_tau_g1.size() < n))
            throw std::invalid_argument("generate_parameters_from_powers_of_tau: the powers hold fewer points than the domain of " +
                                        std::to_string(n) + " reads");
        ProvingKey pk;
        pk.vk.gamma_abc_g1.resize(ni); pk.a_query.resize(nv); pk.b_g1_query.resize(nv); pk.b_g2_query.resize(nv);
        pk.l_query.resize(nv - ni); pk.h_query.resize(QAP::ID == B2G_REDUCTION_LIBSNARK ? n - 1 : n);
        b2g_powers_desc pd;
        memset(&pd, 0, sizeof pd);
        pd.log_size = powers.power;
        pd.tau_g1 = powers.tau_g1.data(); pd.tau_g2 = powers.tau_g2.data(); pd.alpha_tau_g1 = powers.alpha_tau_g1.data();
        pd.beta_tau_g1 = powers.beta_tau_g1.data(); pd.beta_g2 = &powers.beta_g2;
        b2g_setup_out out = {&pk.vk.alpha_g1, &pk.beta_g1, &pk.delta_g1, &pk.vk.beta_g2, &pk.vk.gamma_g2, &pk.vk.delta_g2,
                             pk.vk.gamma_abc_g1.data(), pk.a_query.data(), pk.b_g1_query.data(), pk.b_g2_query.data(),
                             pk.l_query.data(), pk.h_query.data()};
        const Gpu::MatDesc md(matrices, nv, QAP::ID, true);
        if (powers.prepared && n <= (1ull << powers.lagrange.power)) {
            // the Lagrange route (b2g_setup_from_lagrange): blocks log n and log n + 1 must be there, and 2n powers below
            // the prepared power
            const b2g_lagrange_desc ld = lagrange_desc(powers);
            if (powers.lagrange.tau_g1.size() < 4 * n - 1 || powers.lagrange.tau_g2.size() < 2 * n - 1 ||
                powers.lagrange.alpha_tau_g1.size() < 2 * n - 1 || powers.lagrange.beta_tau_g1.size() < 2 * n - 1 ||
                (n < (1ull << powers.lagrange.power) && powers.tau_g1.size() < 2 * n))
                throw std::invalid_argument("generate_parameters_from_powers_of_tau: the Lagrange sections hold fewer points than the "
                                            "domain of " + std::to_string(n) + " reads");
            check(b2g_setup_from_lagrange(gpu.ctx(), &md.d, &pd, &ld, &out));
        } else {
            check(b2g_setup_from_powers(gpu.ctx(), &md.d, &pd, &out));
        }
        return pk;
    }

    // `snarkjs powersoftau prepare phase2` (b2g_powers_prepare): the ceremony of power `power` (0: min(powers.power, 26))
    // formed by the prefix of `powers`, with its Lagrange sections.  Throws std::invalid_argument for a power out of range or
    // vectors shorter than it reads.
    static Powers prepare_powers_of_tau(const Powers& powers, uint32_t power = 0, Gpu& gpu = Gpu::instance()) {
        const uint32_t K = power ? power : std::min<uint32_t>(powers.power, 26);
        if (K < 1 || K > std::min<uint32_t>(powers.power, 26))
            throw std::invalid_argument("prepare_powers_of_tau: power " + std::to_string(K) + " is out of range");
        const size_t n = (size_t)1 << K;
        if (powers.tau_g1.size() < 2 * n - 1 || powers.tau_g2.size() < n || powers.alpha_tau_g1.size() < n || powers.beta_tau_g1.size() < n)
            throw std::invalid_argument("prepare_powers_of_tau: the powers hold fewer points than power " + std::to_string(K) + " reads");
        Powers out;
        out.power = K; out.ceremony_power = powers.ceremony_power;
        out.tau_g1.assign(powers.tau_g1.begin(), powers.tau_g1.begin() + (2 * n - 1));
        out.tau_g2.assign(powers.tau_g2.begin(), powers.tau_g2.begin() + n);
        out.alpha_tau_g1.assign(powers.alpha_tau_g1.begin(), powers.alpha_tau_g1.begin() + n);
        out.beta_tau_g1.assign(powers.beta_tau_g1.begin(), powers.beta_tau_g1.begin() + n);
        out.beta_g2 = powers.beta_g2;
        out.prepared = true;
        out.lagrange.power = K;
        out.lagrange.tau_g1.resize(4 * n - 1); out.lagrange.tau_g2.resize(2 * n - 1);
        out.lagrange.alpha_tau_g1.resize(2 * n - 1); out.lagrange.beta_tau_g1.resize(2 * n - 1);
        b2g_powers_desc pd;
        memset(&pd, 0, sizeof pd);
        pd.log_size = powers.power;
        pd.tau_g1 = out.tau_g1.data(); pd.tau_g2 = out.tau_g2.data(); pd.alpha_tau_g1 = out.alpha_tau_g1.data();
        pd.beta_tau_g1 = out.beta_tau_g1.data(); pd.beta_g2 = &out.beta_g2;
        b2g_lagrange_out od = {K, 0, out.lagrange.tau_g1.data(), out.lagrange.tau_g2.data(), out.lagrange.alpha_tau_g1.data(),
                               out.lagrange.beta_tau_g1.data()};
        check(b2g_powers_prepare(gpu.ctx(), &pd, &od));
        return out;
    }

    // `snarkjs powersoftau contribute` (b2g_powers_contribute): the ceremony of (tau t, alpha a, beta b) from the whole
    // ceremony `powers` of (tau, alpha, beta), the secrets canonical in [1, r); no Lagrange sections (the input's no longer
    // match).  The library's copies of the secrets and the copies made here are wiped.  Throws std::invalid_argument for vectors
    // without the counts of powers.power.
    static Powers contribute_powers_of_tau(const Powers& powers, const BigInt256& t, const BigInt256& a, const BigInt256& b,
                                           Gpu& gpu = Gpu::instance()) {
        const size_t n = (size_t)1 << powers.power;
        if (powers.tau_g1.size() != 2 * n - 1 || powers.tau_g2.size() != n || powers.alpha_tau_g1.size() != n || powers.beta_tau_g1.size() != n)
            throw std::invalid_argument("contribute_powers_of_tau: the powers do not hold the counts of power " + std::to_string(powers.power));
        Powers out;
        out.power = powers.power; out.ceremony_power = powers.ceremony_power;
        out.tau_g1.resize(2 * n - 1); out.tau_g2.resize(n); out.alpha_tau_g1.resize(n); out.beta_tau_g1.resize(n);
        b2g_powers_desc pd;
        memset(&pd, 0, sizeof pd);
        pd.log_size = powers.power;
        pd.tau_g1 = powers.tau_g1.data(); pd.tau_g2 = powers.tau_g2.data(); pd.alpha_tau_g1 = powers.alpha_tau_g1.data();
        pd.beta_tau_g1 = powers.beta_tau_g1.data(); pd.beta_g2 = &powers.beta_g2;
        b2g_powers_out od = {out.tau_g1.data(), out.tau_g2.data(), out.alpha_tau_g1.data(), out.beta_tau_g1.data(), &out.beta_g2};
        BigInt256 sec[3] = {t, a, b};
        const b2g_powers_secrets sd = {sec[0].l, sec[1].l, sec[2].l};
        const int rc = b2g_powers_contribute(gpu.ctx(), &pd, &sd, &od);
        volatile uint64_t* wipe = sec[0].l;
        for (int i = 0; i < 12; i++) wipe[i] = 0;
        check(rc);
        return out;
    }
    // the same with t, a, b drawn from std::random_device by the Fr::rand limb rule, again while zero
    static Powers contribute_powers_of_tau(const Powers& powers, Gpu& gpu = Gpu::instance()) {
        std::random_device rd;
        auto next = [&rd]() { return ((uint64_t)rd() << 32) | rd(); };
        BigInt256 s[3];
        for (BigInt256& x : s) {
            Fr f;
            while (f.is_zero()) f = Fr::rand(next);
            x = f.into_bigint();
            volatile uint64_t* wipe = f.l;
            for (int i = 0; i < 4; i++) wipe[i] = 0;
        }
        struct Wipe { BigInt256* s; ~Wipe() { volatile uint64_t* w = s[0].l; for (int i = 0; i < 12; i++) w[i] = 0; } } guard{s};
        return contribute_powers_of_tau(powers, s[0], s[1], s[2], gpu);
    }

    // the algebraic checks of `snarkjs powersoftau verify` (b2g_powers_check): whether the prefix a domain of 2^log_n points
    // reads (log_n = 0: the ceremony's power) holds powers of one tau with the same alpha and beta on the standard generators.
    // The challenges come from std::random_device, drawn after the powers are fixed, unless five are given (canonical, in
    // [1, r)).  Throws std::invalid_argument when log_n exceeds the power or the vectors hold fewer points than it reads.
    static PowersCheck verify_powers_of_tau(const Powers& powers, uint32_t log_n = 0, Gpu& gpu = Gpu::instance(),
                                            const std::vector<BigInt256>* challenges = nullptr) {
        if (!log_n) log_n = powers.power;
        if (log_n > powers.power) throw std::invalid_argument("verify_powers_of_tau: log_n exceeds the ceremony's power");
        const size_t n = (size_t)1 << log_n;
        if (powers.tau_g1.size() < 2 * n - 1 || powers.tau_g2.size() < n || powers.alpha_tau_g1.size() < n || powers.beta_tau_g1.size() < n)
            throw std::invalid_argument("verify_powers_of_tau: the powers hold fewer points than a domain of " + std::to_string(n) + " reads");
        std::vector<BigInt256> drawn = challenges ? *challenges : powers_challenges();
        if (drawn.size() != 5 && drawn.size() != 6)
            throw std::invalid_argument("verify_powers_of_tau: five challenges (rho, sigma, pi, kappa, eps) and an optional sixth");
        if (powers.prepared && drawn.size() == 5) drawn.push_back(powers_challenges()[0]);  // the Lagrange check's rho
        b2g_powers_desc pd;
        memset(&pd, 0, sizeof pd);
        pd.log_size = powers.power;
        pd.tau_g1 = powers.tau_g1.data(); pd.tau_g2 = powers.tau_g2.data(); pd.alpha_tau_g1 = powers.alpha_tau_g1.data();
        pd.beta_tau_g1 = powers.beta_tau_g1.data(); pd.beta_g2 = &powers.beta_g2;
        b2g_powers_report rep;
        check(b2g_powers_check(gpu.ctx(), &pd, log_n, drawn.data(), &rep));
        if (rep.ok && powers.prepared) {
            // the Lagrange sections up to log_n (b2g_lagrange_check), with the sixth challenge
            if (log_n > powers.lagrange.power || powers.lagrange.tau_g1.size() < 4 * n - 1 || powers.lagrange.tau_g2.size() < 2 * n - 1 ||
                powers.lagrange.alpha_tau_g1.size() < 2 * n - 1 || powers.lagrange.beta_tau_g1.size() < 2 * n - 1 ||
                (log_n < powers.lagrange.power && powers.tau_g1.size() < 2 * n))
                throw std::invalid_argument("verify_powers_of_tau: the Lagrange sections hold fewer points than a domain of " +
                                            std::to_string(n) + " reads");
            const b2g_lagrange_desc ld = lagrange_desc(powers);
            check(b2g_lagrange_check(gpu.ctx(), &pd, &ld, log_n, &drawn[5], &rep));
        }
        static const char* const arrays[9] = {"tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2", "lagrange_tau_g1",
                                              "lagrange_tau_g2", "lagrange_alpha_tau_g1", "lagrange_beta_tau_g1"};
        PowersCheck r;
        r.ok = rep.ok != 0;
        r.rule = rep.rule;
        if (!r.ok && rep.rule != 6) { r.array = arrays[rep.array]; r.index = rep.index; }
        return r;
    }

    static b2g_lagrange_desc lagrange_desc(const Powers& p) {
        return b2g_lagrange_desc{p.lagrange.power, 0, p.lagrange.tau_g1.data(), p.lagrange.tau_g2.data(), p.lagrange.alpha_tau_g1.data(),
                                 p.lagrange.beta_tau_g1.data()};
    }

    // `snarkjs zkey verify circuit.r1cs pot.ptau circuit.zkey` without its transcript (b2g_setup_check): whether pk is the key
    // generate_parameters_from_powers_of_tau makes from the matrices (with C) and the ceremony, followed by any chain of
    // contribute calls.  zkey_matrices, the matrices read_zkey returns with the key, must then hold the circuit's A and B
    // (compared row by row in canonical form) and its counts.  The challenges rho and sigma come from std::random_device, drawn
    // after the key is fixed, unless two are given (canonical, in [1, r)).  Throws std::invalid_argument when the powers hold
    // fewer points than the circuit's domain reads.
    static SetupCheck verify_proving_key(const ConstraintMatrices& matrices, const Powers& powers, const ProvingKey& pk,
                                         const ConstraintMatrices* zkey_matrices = nullptr, Gpu& gpu = Gpu::instance(),
                                         const std::vector<BigInt256>* challenges = nullptr) {
        const size_t ni = matrices.num_instance_variables, nv = ni + matrices.num_witness_variables, m = matrices.num_constraints;
        if (ni == 0) throw SynthesisError("verify_proving_key: no instance variable");
        if (m && matrices.c.empty()) throw SynthesisError("verify_proving_key needs the C matrix (R1CS route); zkey matrices have none");
        SetupCheck r;
        if (zkey_matrices) {
            const ConstraintMatrices& z = *zkey_matrices;
            const size_t have[3] = {z.num_instance_variables, z.num_constraints, z.num_instance_variables + z.num_witness_variables};
            const size_t want[3] = {ni, m, nv};
            static const char* const what[3] = {"num_inputs", "num_constraints", "n_vars"};
            for (int k = 0; k < 3; k++)
                if (have[k] != want[k]) {
                    r.why = std::string("the matrices' ") + what[k] + " " + std::to_string(have[k]) + " differs from the circuit's " + std::to_string(want[k]);
                    return r;
                }
            const std::pair<const Matrix*, const Matrix*> mats[2] = {{&z.a, &matrices.a}, {&z.b, &matrices.b}};
            for (int k = 0; k < 2; k++) {
                const auto got = detail::canonical_rows(*mats[k].first, m), want_rows = detail::canonical_rows(*mats[k].second, m);
                for (size_t row = 0; row < m; row++) {
                    bool same = got[row].size() == want_rows[row].size();
                    for (size_t e = 0; same && e < got[row].size(); e++)
                        same = got[row][e].first == want_rows[row][e].first && got[row][e].second == want_rows[row][e].second;
                    if (!same) { r.why = std::string("matrix ") + (k ? "B" : "A") + " differs from the circuit at row " + std::to_string(row); return r; }
                }
            }
        }
        size_t n = 1;
        while (n < m + ni) n <<= 1;
        const size_t nh = QAP::ID == B2G_REDUCTION_LIBSNARK ? n - 1 : n;
        const std::pair<const char*, std::pair<size_t, size_t>> shapes[6] = {
            {"gamma_abc_g1", {pk.vk.gamma_abc_g1.size(), ni}}, {"a_query", {pk.a_query.size(), nv}}, {"b_g1_query", {pk.b_g1_query.size(), nv}},
            {"b_g2_query", {pk.b_g2_query.size(), nv}}, {"l_query", {pk.l_query.size(), nv - ni}}, {"h_query", {pk.h_query.size(), nh}}};
        for (const auto& sh : shapes)
            if (sh.second.first != sh.second.second) {
                r.why = std::string(sh.first) + " holds " + std::to_string(sh.second.first) + " points; " +
                        (std::string(sh.first) == "h_query" ? std::string("a ") + (QAP::ID == B2G_REDUCTION_LIBSNARK ? "LibsnarkReduction" : "CircomReduction") +
                                                                  " domain of " + std::to_string(n) + " needs "
                                                            : std::string("the circuit needs ")) + std::to_string(sh.second.second);
                return r;
            }
        if (n <= (1ull << powers.power) &&
            (powers.tau_g1.size() < 2 * n - 1 || powers.tau_g2.size() < n || powers.alpha_tau_g1.size() < n || powers.beta_tau_g1.size() < n))
            throw std::invalid_argument("verify_proving_key: the powers hold fewer points than the domain of " + std::to_string(n) + " reads");
        const std::vector<BigInt256> drawn = challenges ? *challenges : powers_challenges(2);
        if (drawn.size() != 2) throw std::invalid_argument("verify_proving_key: two challenges (rho, sigma)");
        b2g_powers_desc pd;
        memset(&pd, 0, sizeof pd);
        pd.log_size = powers.power;
        pd.tau_g1 = powers.tau_g1.data(); pd.tau_g2 = powers.tau_g2.data(); pd.alpha_tau_g1 = powers.alpha_tau_g1.data();
        pd.beta_tau_g1 = powers.beta_tau_g1.data(); pd.beta_g2 = &powers.beta_g2;
        b2g_key_desc kd;
        memset(&kd, 0, sizeof kd);
        kd.n_vars = (uint32_t)nv; kd.n_ic = (uint32_t)ni; kd.n_l = (uint32_t)(nv - ni); kd.n_h = (uint32_t)nh;
        kd.alpha_g1 = &pk.vk.alpha_g1; kd.beta_g1 = &pk.beta_g1; kd.delta_g1 = &pk.delta_g1;
        kd.beta_g2 = &pk.vk.beta_g2; kd.gamma_g2 = &pk.vk.gamma_g2; kd.delta_g2 = &pk.vk.delta_g2;
        kd.gamma_abc_g1 = pk.vk.gamma_abc_g1.data(); kd.a_query = pk.a_query.data(); kd.b_g1_query = pk.b_g1_query.data();
        kd.b_g2_query = pk.b_g2_query.data(); kd.l_query = pk.l_query.empty() ? nullptr : pk.l_query.data(); kd.h_query = pk.h_query.data();
        const Gpu::MatDesc md(matrices, nv, QAP::ID, true);
        b2g_setup_report rep;
        check(b2g_setup_check(gpu.ctx(), &md.d, &pd, &kd, drawn.data(), &rep));
        r.ok = rep.ok != 0;
        if (r.ok) return r;
        static const char* const fields[12] = {"alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1",
                                               "a_query", "b_g1_query", "b_g2_query", "l_query", "h_query"};
        static const char* const arrays[5] = {"tau_g1", "tau_g2", "alpha_tau_g1", "beta_tau_g1", "beta_g2"};
        const std::string name = rep.side ? arrays[rep.field % 5] : fields[rep.field % 12];
        if (rep.rule == 8) {
            if (rep.field == 6) r.why = "gamma_abc_g1 / l_query do not match the circuit and ceremony";
            else if (rep.field == 2) r.why = "delta_g1 and delta_g2 disagree";
            else r.why = name + " does not match the circuit and ceremony";
        } else if (rep.rule == 7) {
            r.why = name + " is not the ceremony's";
        } else {
            const bool g2 = name == "beta_g2" || name == "gamma_g2" || name == "delta_g2" || name == "b_g2_query" || name == "tau_g2";
            static const char* const texts[5] = {"", "a coordinate >= p", "off the curve", "at infinity", "not in G2"};
            r.why = name + "[" + std::to_string(rep.index) + "]: " + (rep.rule == 2 && g2 ? "off the twist" : rep.rule < 5 ? texts[rep.rule] : "?");
        }
        return r;
    }

    // `snarkjs zkey contribute` (b2g_delta_update): pk with delta multiplied by x (nonzero, below r) and the L and H queries
    // divided by it; the library's copies of x are wiped
    static ProvingKey contribute(const ProvingKey& pk, const Fr& x, Gpu& gpu = Gpu::instance()) {
        ProvingKey out;
        out.vk = pk.vk; out.beta_g1 = pk.beta_g1; out.a_query = pk.a_query; out.b_g1_query = pk.b_g1_query;
        out.b_g2_query = pk.b_g2_query;
        out.l_query.resize(pk.l_query.size()); out.h_query.resize(pk.h_query.size());
        b2g_delta_key before = delta_key(pk), after = delta_key(out);
        BigInt256 xb = x.into_bigint();
        const int rc = b2g_delta_update(gpu.ctx(), &before, xb.l, &after);
        volatile uint64_t* wipe = xb.l;
        for (int i = 0; i < 4; i++) wipe[i] = 0;
        check(rc);
        return out;
    }
    // the same with x = Fr::rand(rng), drawn again while zero (an Fr argument selects the call above)
    template <class Rng, class = typename std::enable_if<!std::is_same<Rng, Fr>::value>::type>
    static ProvingKey contribute(const ProvingKey& pk, Rng& rng, Gpu& gpu = Gpu::instance()) {
        Fr x;
        while (x.is_zero()) x = Fr::rand(rng);
        const ProvingKey out = contribute(pk, x, gpu);
        volatile uint64_t* wipe = x.l;
        for (int i = 0; i < 4; i++) wipe[i] = 0;
        return out;
    }

    // the delta checks of `snarkjs zkey verify` (b2g_delta_update_check, weights from std::random_device): whether `after`
    // is `before` with one or more contributions.  The fields a contribution leaves alone are compared on the host.
    static bool verify_contribution(const ProvingKey& before, const ProvingKey& after, Gpu& gpu = Gpu::instance()) {
        auto same = [](const void* a, const void* b, size_t bytes) { return !memcmp(a, b, bytes); };
        auto same_vec = [&](const auto& a, const auto& b) {
            return a.size() == b.size() && (a.empty() || same(a.data(), b.data(), a.size() * sizeof(a[0])));
        };
        if (!same(&before.vk.alpha_g1, &after.vk.alpha_g1, 64) || !same(&before.beta_g1, &after.beta_g1, 64) ||
            !same(&before.vk.beta_g2, &after.vk.beta_g2, 128) || !same(&before.vk.gamma_g2, &after.vk.gamma_g2, 128) ||
            !same_vec(before.vk.gamma_abc_g1, after.vk.gamma_abc_g1) || !same_vec(before.a_query, after.a_query) ||
            !same_vec(before.b_g1_query, after.b_g1_query) || !same_vec(before.b_g2_query, after.b_g2_query) ||
            before.l_query.size() != after.l_query.size() || before.h_query.size() != after.h_query.size())
            return false;
        b2g_delta_key b = delta_key(before), a = delta_key(after);
        const std::vector<uint32_t> w = batch_weights(before.l_query.size() + before.h_query.size());
        uint8_t verdict = 0;
        check(b2g_delta_update_check(gpu.ctx(), &b, &a, w.data(), &verdict));
        return verdict != 0;
    }

    // Groth16::generate_random_parameters_with_reduction(circuit, rng): alpha, beta, gamma, delta, tau drawn with Fr::rand in that
    // order, on the standard generators
    template <class Rng>
    static ProvingKey generate_random_parameters_with_reduction(const ConstraintMatrices& matrices, Rng& rng, Gpu& gpu = Gpu::instance()) {
        const Fr alpha = Fr::rand(rng), beta = Fr::rand(rng), gamma = Fr::rand(rng), delta = Fr::rand(rng), tau = Fr::rand(rng);
        return generate_parameters_with_qap(matrices, alpha, beta, gamma, delta, nullptr, nullptr, tau, gpu);
    }

    template <class Rng>
    static Proof prove(const ProvingKey& pk, const ConstraintMatrices& matrices, const std::vector<Fr>& full_assignment, Rng& rng,
                       Gpu& gpu = Gpu::instance()) {
        Fr r = Fr::rand(rng), s = Fr::rand(rng);        // r first, then s (create_random_proof_with_reduction)
        return create_proof_with_reduction_and_matrices(pk, r, s, matrices, matrices.num_instance_variables, matrices.num_constraints,
                                                        full_assignment, gpu);
    }
};

typedef Groth16T<CircomReduction> Groth16;

// ---------------------------------------------------------------------------------------------- R1CS route (host)
// R1CSFile / R1CS: /root/reference/src/circom/r1cs_reader.rs:54-249; to_matrices = what CircomCircuit::generate_constraints
// + ConstraintSystem::to_matrices yield (src/circom/circuit.rs:30-82: column index = wire index).
struct R1CS {
    size_t num_inputs = 0, num_aux = 0, num_variables = 0;
    struct Constraint { std::vector<std::pair<size_t, Fr>> a, b, c; };          // (index, coeff): src/circom/mod.rs:13-14
    std::vector<Constraint> constraints;
    std::vector<uint64_t> wire_mapping;

    static R1CS read(std::istream& r) {
        char magic[4]; detail::read_exact(r, magic, 4);
        if (memcmp(magic, "r1cs", 4)) throw SerializationError("Invalid magic number");
        if (detail::read_le<uint32_t>(r) != 1) throw SerializationError("Unsupported version");
        uint32_t nsec = detail::read_le<uint32_t>(r);
        std::map<uint32_t, std::pair<uint64_t, uint64_t>> sec;
        for (uint32_t i = 0; i < nsec; i++) {
            uint32_t t = detail::read_le<uint32_t>(r); uint64_t sz = detail::read_le<uint64_t>(r);
            sec[t] = {(uint64_t)r.tellg(), sz};
            r.seekg((std::streamoff)sz, std::ios::cur);
        }
        for (uint32_t t : {1u, 2u, 3u}) if (!sec.count(t)) throw SerializationError("missing r1cs section");
        r.clear(); r.seekg((std::streamoff)sec[1].first);
        if (detail::read_le<uint32_t>(r) != 32) throw SerializationError("This parser only supports 32-byte fields");
        uint64_t prime[4]; detail::read_exact(r, prime, 32);
        if (memcmp(prime, detail::FR_P, 32)) throw SerializationError("This parser only supports bn256");
        uint32_t n_wires = detail::read_le<uint32_t>(r), n_pub_out = detail::read_le<uint32_t>(r), n_pub_in = detail::read_le<uint32_t>(r);
        detail::read_le<uint32_t>(r); detail::read_le<uint64_t>(r);
        uint32_t n_cons = detail::read_le<uint32_t>(r);
        R1CS out;
        out.num_inputs = 1 + n_pub_in + n_pub_out; out.num_variables = n_wires; out.num_aux = n_wires - out.num_inputs;
        r.seekg((std::streamoff)sec[2].first);
        auto lc = [&](std::vector<std::pair<size_t, Fr>>& v) {
            uint32_t n = detail::read_le<uint32_t>(r);
            for (uint32_t k = 0; k < n; k++) { uint32_t w = detail::read_le<uint32_t>(r); BigInt256 b; detail::read_exact(r, b.l, 32); v.push_back({w, Fr::from_bigint(b)}); }
        };
        out.constraints.resize(n_cons);
        for (auto& c : out.constraints) { lc(c.a); lc(c.b); lc(c.c); }
        if (sec[3].second != (uint64_t)n_wires * 8) throw SerializationError("Invalid map section size");
        r.seekg((std::streamoff)sec[3].first);
        out.wire_mapping.resize(n_wires);
        if (n_wires) detail::read_exact(r, out.wire_mapping.data(), (size_t)n_wires * 8);
        if (n_wires && out.wire_mapping[0] != 0) throw SerializationError("Wire 0 should always be mapped to 0");
        return out;
    }

    ConstraintMatrices to_matrices() const {
        ConstraintMatrices m;
        m.num_instance_variables = num_inputs; m.num_witness_variables = num_aux; m.num_constraints = constraints.size();
        m.a.resize(constraints.size()); m.b.resize(constraints.size()); m.c.resize(constraints.size());
        for (size_t i = 0; i < constraints.size(); i++) {
            for (auto& e : constraints[i].a) m.a[i].push_back({e.second, e.first});
            for (auto& e : constraints[i].b) m.b[i].push_back({e.second, e.first});
            for (auto& e : constraints[i].c) m.c[i].push_back({e.second, e.first});
            m.a_num_non_zero += m.a[i].size(); m.b_num_non_zero += m.b[i].size(); m.c_num_non_zero += m.c[i].size();
        }
        return m;
    }
};

// ---------------------------------------------------------------------------------------------- ark-serialize keys
// serialize_proving_key / serialize_verifying_key    <- pk.serialize_compressed(&mut w) / serialize_uncompressed (ark-serialize 0.5)
// deserialize_proving_key / deserialize_verifying_key <- ProvingKey / VerifyingKey::<Bn254>::deserialize_compressed(&mut r) /
//                                                      deserialize_uncompressed (Validate::Yes)
// deserialize_verifying_keys                          <- the same for many keys, decoded in two device calls
// The layout is ark_serialize.py's (fields in declaration order, h_query before l_query, a Vec = u64 length then its
// elements); the host parses lengths only, and every point is encoded or decoded on the device (b2g_points_serialize /
// b2g_points_deserialize): all G1 points of a call in one device call, all G2 points in one more.  A refusal throws
// SerializationError naming the field and index ("b_g2_query[17]: ...").
namespace detail {
struct KeyField { const char* name; bool vec, g2; };
static const KeyField VK_FIELDS[] = {{"alpha_g1", false, false}, {"beta_g2", false, true}, {"gamma_g2", false, true},
                                     {"delta_g2", false, true}, {"gamma_abc_g1", true, false}};
static const KeyField PK_FIELDS[] = {{"alpha_g1", false, false}, {"beta_g2", false, true}, {"gamma_g2", false, true},
                                     {"delta_g2", false, true}, {"gamma_abc_g1", true, false}, {"beta_g1", false, false},
                                     {"delta_g1", false, false}, {"a_query", true, false}, {"b_g1_query", true, false},
                                     {"b_g2_query", true, true}, {"h_query", true, false}, {"l_query", true, false}};
inline size_t point_size(bool g2, bool compress) { return (g2 ? 64 : 32) * (compress ? 1 : 2); }

// the points of one field of one key: Montgomery rows (on write) or serialized bytes (on read), and their number
struct FieldPoints { const KeyField* f; const uint8_t* data; size_t count; };

inline std::vector<FieldPoints> vk_points(const VerifyingKey& vk) {
    return {{&VK_FIELDS[0], (const uint8_t*)&vk.alpha_g1, 1}, {&VK_FIELDS[1], (const uint8_t*)&vk.beta_g2, 1},
            {&VK_FIELDS[2], (const uint8_t*)&vk.gamma_g2, 1}, {&VK_FIELDS[3], (const uint8_t*)&vk.delta_g2, 1},
            {&VK_FIELDS[4], (const uint8_t*)vk.gamma_abc_g1.data(), vk.gamma_abc_g1.size()}};
}

inline std::vector<uint8_t> encode_key(const std::vector<FieldPoints>& fields, bool compress, int device) {
    std::vector<uint8_t> enc[2];
    for (int g2 = 0; g2 < 2; g2++) {
        std::vector<uint8_t> pts;
        for (const FieldPoints& fp : fields) if (fp.f->g2 == (bool)g2) pts.insert(pts.end(), fp.data, fp.data + fp.count * (g2 ? 128 : 64));
        const size_t n = pts.size() / (g2 ? 128 : 64);
        enc[g2].resize(n * point_size(g2, compress));
        if (n) check(b2g_points_serialize(Gpu::on(device).ctx(), g2, compress, n, pts.data(), enc[g2].data()));
    }
    std::vector<uint8_t> out;
    size_t at[2] = {0, 0};
    for (const FieldPoints& fp : fields) {
        const int g2 = fp.f->g2;
        if (fp.f->vec) { const uint64_t c = fp.count; const uint8_t* b = (const uint8_t*)&c; out.insert(out.end(), b, b + 8); }
        const size_t bytes = fp.count * point_size(g2, compress);
        out.insert(out.end(), enc[g2].begin() + at[g2], enc[g2].begin() + at[g2] + bytes);
        at[g2] += bytes;
    }
    return out;
}

// the serialized points of every field, length prefixes parsed; the input is read in chunks, so a huge length prefix
// never allocates its size
inline std::vector<std::pair<uint64_t, std::vector<uint8_t>>> parse_key(std::istream& r, const KeyField* fields, size_t n_fields,
                                                                       bool compress, const std::string& at) {
    std::vector<std::pair<uint64_t, std::vector<uint8_t>>> out;
    for (size_t k = 0; k < n_fields; k++) {
        const KeyField& f = fields[k];
        uint64_t count = 1;
        if (f.vec) {
            r.read(reinterpret_cast<char*>(&count), 8);
            if (r.gcount() != 8) throw SerializationError(at + f.name + ": the input ends in the length");
        }
        const size_t size = point_size(f.g2, compress);
        std::vector<uint8_t> raw;
        for (uint64_t left = count; left;) {
            const uint64_t m = std::min<uint64_t>(left, (1u << 26) / size);
            const size_t have = raw.size();
            raw.resize(have + m * size);
            r.read(reinterpret_cast<char*>(raw.data() + have), (std::streamsize)(m * size));
            if ((size_t)r.gcount() != m * size) throw SerializationError(at + f.name + ": the input ends before its " + std::to_string(count) + " points");
            left -= m;
        }
        out.push_back({count, std::move(raw)});
    }
    return out;
}

// decodes the points of every key (keys[k][field] from parse_key) in two device calls: decoded[k][field] = Montgomery rows.
// The refused point that comes first in serialized order throws.
inline std::vector<std::vector<std::vector<uint8_t>>> decode_keys(const std::vector<std::vector<std::pair<uint64_t, std::vector<uint8_t>>>>& keys,
                                                                  const KeyField* fields, size_t n_fields, bool compress,
                                                                  const std::vector<std::string>& ats, int device) {
    std::vector<std::vector<std::vector<uint8_t>>> out(keys.size(), std::vector<std::vector<uint8_t>>(n_fields));
    std::tuple<size_t, size_t, uint64_t> first_bad{SIZE_MAX, 0, 0};
    for (int g2 = 0; g2 < 2; g2++) {
        std::vector<uint8_t> raw;
        size_t n = 0;
        for (const auto& key : keys)
            for (size_t f = 0; f < n_fields; f++)
                if (fields[f].g2 == (bool)g2) { raw.insert(raw.end(), key[f].second.begin(), key[f].second.end()); n += key[f].first; }
        if (!n) continue;
        const size_t row = g2 ? 128 : 64;
        std::vector<uint8_t> pts(n * row);
        uint64_t bad = n;
        check(b2g_points_deserialize(Gpu::on(device).ctx(), g2, compress, n, raw.data(), pts.data(), &bad));
        size_t o = 0;
        for (size_t k = 0; k < keys.size(); k++)
            for (size_t f = 0; f < n_fields; f++) {
                if (fields[f].g2 != (bool)g2) continue;
                const uint64_t c = keys[k][f].first;
                if (bad >= o && bad < o + c) first_bad = std::min(first_bad, std::make_tuple(k, f, bad - o));
                out[k][f].assign(pts.begin() + o * row, pts.begin() + (o + c) * row);
                o += c;
            }
    }
    if (std::get<0>(first_bad) != SIZE_MAX) {
        const auto [k, f, i] = first_bad;
        throw SerializationError(ats[k] + fields[f].name + (fields[f].vec ? "[" + std::to_string(i) + "]" : std::string()) +
                                 ": not a valid " + (compress ? "compressed " : "uncompressed ") + (fields[f].g2 ? "G2" : "G1") + " point (Validate::Yes)");
    }
    return out;
}

template <class T> inline void rows_into(T& dst, const std::vector<uint8_t>& rows) { memcpy(&dst, rows.data(), sizeof(T)); }
template <class T> inline void rows_into(std::vector<T>& dst, const std::vector<uint8_t>& rows) {
    dst.resize(rows.size() / sizeof(T));
    if (!dst.empty()) memcpy(dst.data(), rows.data(), rows.size());
}

inline VerifyingKey vk_from(const std::vector<std::vector<uint8_t>>& d) {
    VerifyingKey vk;
    rows_into(vk.alpha_g1, d[0]); rows_into(vk.beta_g2, d[1]); rows_into(vk.gamma_g2, d[2]); rows_into(vk.delta_g2, d[3]);
    rows_into(vk.gamma_abc_g1, d[4]);
    return vk;
}

inline void check_gamma_abc(uint64_t count, const std::string& at) {
    if (count == 0) throw SerializationError(at + "gamma_abc_g1: empty (a key has at least the constant term's point)");
}
}  // namespace detail

inline std::vector<uint8_t> serialize_verifying_key(const VerifyingKey& vk, bool compress = true, int device = 0) {
    return detail::encode_key(detail::vk_points(vk), compress, device);
}

inline std::vector<uint8_t> serialize_proving_key(const ProvingKey& pk, bool compress = true, int device = 0) {
    std::vector<detail::FieldPoints> f = detail::vk_points(pk.vk);
    const detail::KeyField* F = detail::PK_FIELDS;
    f.push_back({&F[5], (const uint8_t*)&pk.beta_g1, 1});
    f.push_back({&F[6], (const uint8_t*)&pk.delta_g1, 1});
    f.push_back({&F[7], (const uint8_t*)pk.a_query.data(), pk.a_query.size()});
    f.push_back({&F[8], (const uint8_t*)pk.b_g1_query.data(), pk.b_g1_query.size()});
    f.push_back({&F[9], (const uint8_t*)pk.b_g2_query.data(), pk.b_g2_query.size()});
    f.push_back({&F[10], (const uint8_t*)pk.h_query.data(), pk.h_query.size()});
    f.push_back({&F[11], (const uint8_t*)pk.l_query.data(), pk.l_query.size()});
    return detail::encode_key(f, compress, device);
}

// the reader is left just past the key; gamma_abc_g1 must hold at least one point
inline VerifyingKey deserialize_verifying_key(std::istream& r, bool compress = true, int device = 0) {
    auto key = detail::parse_key(r, detail::VK_FIELDS, 5, compress, "");
    detail::check_gamma_abc(key[4].first, "");
    return detail::vk_from(detail::decode_keys({key}, detail::VK_FIELDS, 5, compress, {""}, device)[0]);
}

// many keys, every G1 point in one device call and every G2 point in one more; a refusal names the key ("key 3: ...")
inline std::vector<VerifyingKey> deserialize_verifying_keys(const std::vector<std::vector<uint8_t>>& blobs, bool compress = true, int device = 0) {
    std::vector<std::vector<std::pair<uint64_t, std::vector<uint8_t>>>> keys;
    std::vector<std::string> ats;
    for (size_t k = 0; k < blobs.size(); k++) {
        std::istringstream r(std::string(blobs[k].begin(), blobs[k].end()));
        ats.push_back("key " + std::to_string(k) + ": ");
        keys.push_back(detail::parse_key(r, detail::VK_FIELDS, 5, compress, ats.back()));
        detail::check_gamma_abc(keys.back()[4].first, ats.back());
    }
    std::vector<VerifyingKey> out;
    if (keys.empty()) return out;
    for (const auto& d : detail::decode_keys(keys, detail::VK_FIELDS, 5, compress, ats, device)) out.push_back(detail::vk_from(d));
    return out;
}

// the reader is left just past the key.  Keys whose vector lengths disagree (b_g1_query or b_g2_query not of a_query's
// length, l_query not of len(a_query) - len(gamma_abc_g1) points, an empty gamma_abc_g1) are refused although arkworks
// reads them: no proof can be made with such a key.  The key carries no reduction; it proves under the one the caller picks.
inline ProvingKey deserialize_proving_key(std::istream& r, bool compress = true, int device = 0) {
    auto key = detail::parse_key(r, detail::PK_FIELDS, 12, compress, "");
    detail::check_gamma_abc(key[4].first, "");
    const uint64_t n_vars = key[7].first, n_ic = key[4].first;
    if (n_ic > n_vars) throw SerializationError("gamma_abc_g1: " + std::to_string(n_ic) + " points, more than a_query's " + std::to_string(n_vars));
    const std::pair<size_t, uint64_t> want[] = {{8, n_vars}, {9, n_vars}, {11, n_vars - n_ic}};
    for (const auto& [f, n] : want)
        if (key[f].first != n)
            throw SerializationError(std::string(detail::PK_FIELDS[f].name) + ": " + std::to_string(key[f].first) +
                                     " points, the key's a_query and gamma_abc_g1 need " + std::to_string(n));
    const auto d = detail::decode_keys({key}, detail::PK_FIELDS, 12, compress, {""}, device)[0];
    ProvingKey pk;
    pk.vk = detail::vk_from(d);
    detail::rows_into(pk.beta_g1, d[5]); detail::rows_into(pk.delta_g1, d[6]);
    detail::rows_into(pk.a_query, d[7]); detail::rows_into(pk.b_g1_query, d[8]); detail::rows_into(pk.b_g2_query, d[9]);
    detail::rows_into(pk.h_query, d[10]); detail::rows_into(pk.l_query, d[11]);
    return pk;
}

}  // namespace ark_circom
