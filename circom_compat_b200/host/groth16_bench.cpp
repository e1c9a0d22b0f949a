// groth16_bench.cpp - C++ counterpart of /root/reference/benches/groth16.rs:13-85: read a zkey, obtain the full assignment,
// draw / take (r, s), call Groth16::create_proof_with_reduction_and_matrices repeatedly and report the time per proof.
//
//   groth16_bench --parse-only <circuit.zkey> [--dump-key]         host-only: print what read_zkey produced (no GPU)
//   groth16_bench --verify <circuit.zkey> <proof_hex> [inputs...]  host-only: process_vk + verify_with_processed_vk
//   groth16_bench --ethereum <circuit.zkey> <proof_hex> [inputs...] host-only: src/ethereum.rs views of vk / proof / inputs, both directions,
//                                                                   and the proof's ark-serialize compressed bytes
//   groth16_bench <circuit.zkey> chain:<a>|<witness.wtns> [iters] [r_hex s_hex]
//       B2G_MANY=K: also K proofs in one device pass (Groth16::create_proofs)
//       B2G_PROVE_KEYS=K: also load K copies of the key as one group (Groth16::load_proving_keys) and prove one proof of
//       chain:<a + k> under copy k, all in one device pass (Groth16::create_proofs_keys), timing the keyed call
//       B2G_VERIFY_MANY=K: also prove K proofs, negate A in every other one, and compare Groth16::verify_many's verdicts with
//       verify_with_processed_vk called per proof (timing both)
//       B2G_VERIFY_BATCH=K: also prove K proofs and compare Groth16::verify_batch's verdict, on them and with the last
//       proof's A negated, with verify_with_processed_vk over every proof (timing the batch call)
//       B2G_VERIFY_COMPRESSED=K: also prove K proofs, serialize them compressed, flip the sign bit of A in every other one,
//       compare Groth16::verify_many_compressed's verdicts with the host verifier, decode the untouched ones back, and print
//       Groth16::verify_batch_compressed's verdict on the untouched and on the flipped set
//       B2G_VERIFY_LOCATE=K: also prove K proofs, negate A in proofs 0, K / 2 and K - 1, and compare
//       Groth16::verify_batch_locate's verdicts with verify_with_processed_vk called per proof (timing the locate call)
//       B2G_VERIFY_KEYS=K: also prove K proofs, split them into up to four batches of the key plus an empty one, negate A in
//       the last proof of the second batch, and compare Groth16::verify_batch_keys's verdicts with the host verifier per
//       batch (timing the keyed call)
//       B2G_LOAD_KEYS=K: also prove K proofs, prepare K copies of the key on the device with Groth16::load_verifying_keys,
//       negate A in every third proof, and compare Groth16::verify_batch_keys's verdicts (proof i under copy i) with the host
//       verifier, printing the launches of both calls
//       B2G_VERIFY_KEYS_LOCATE=K: also prove K proofs, split them into up to four batches of the key with an empty one after
//       the first, negate A in the first proof of the first batch, the last proof of the others and proofs 63 and 64 of each
//       batch that has them, and compare Groth16::verify_batch_keys_locate's verdicts with the host verifier per proof
//       (timing the keyed locate call)
//       B2G_RERANDOMIZE=K: also prove K proofs, rerandomize them with Groth16::rerandomize_many (factors from std::mt19937_64
//       seeded with 0x5EED), print every input and output row in hex, and check the outputs with the host verifier
//       B2G_ARK_KEYS=path: also write the key with serialize_proving_key, compressed to path.compressed and uncompressed to
//       path.uncompressed, read each back with deserialize_proving_key, and print its size, its FNV-1a digest and whether
//       the key read back is identical
//   B2G_SETUP=<seed> groth16_bench <circuit.r1cs> <witness.wtns>
//       tests/groth16.rs:75-105 in C++: draw the toxic waste with std::mt19937_64(seed), make the key with
//       Groth16T<LibsnarkReduction>::generate_random_parameters_with_reduction (b2g_setup), print the five secrets, the key
//       (serialize_proving_key, compressed, hex), the proof of the witness under the same rng and the host verifier's verdict
//   B2G_SETUP_PTAU=<file.ptau> groth16_bench <circuit.r1cs> <witness.wtns> [seed]
//       the same flow with a powers-of-tau ceremony in place of the toxic waste (CircomReduction, as snarkjs): read the prefix
//       of the ceremony the circuit needs (read_ptau), make the key (generate_parameters_from_powers_of_tau), apply one
//       contribution with x = Fr::rand(std::mt19937_64(seed)) (default seed 0x5E7), check it (verify_contribution), prove the
//       witness under the same rng and verify on the host; print x, the contributed key (serialize_proving_key, compressed,
//       hex), the check's verdict, the proof and the host verifier's verdict
//   B2G_ZKEY_VERIFY=<file.ptau> groth16_bench <circuit.r1cs> <circuit.zkey>
//       check the key against the circuit and the ceremony with Groth16T::verify_proving_key (CircomReduction, as snarkjs) and
//       print key=1, or key=0 and the reason, and the time of the check in ms (the file reads not included)
//   B2G_PTAU_PREPARE=<in.ptau> groth16_bench <out.ptau> [power]
//       prepare the ceremony (or the one of the given power formed by its prefix) for phase 2 with
//       Groth16T::prepare_powers_of_tau and write it with its Lagrange sections 12-15; prints the power and the time in ms
//   B2G_PTAU_CONTRIBUTE=<in.ptau> groth16_bench <out.ptau> [tau alpha beta]
//       one phase-1 contribution to the whole ceremony with Groth16T::contribute_powers_of_tau, the secrets drawn from
//       std::random_device unless given (decimal, in [1, r)); writes the file and prints the power and the time in ms
//   B2G_PTAU_CHECK=<file.ptau> groth16_bench [log_n]
//       check the ceremony (or the prefix a domain of 2^log_n points reads) with Groth16T::verify_powers_of_tau and print
//       powers=1 or powers=0 with the reason, and the time of the check in ms (the file read not included)
//       chain:<a> = the witness of the reference's squaring-chain bench family for input a
//       (test-vectors/complex-circuit/input.json has a = 3), computed on the host instead of by WASM.
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstdio>
#include <fstream>
#include <iostream>

#include "ark_circom_b200.hpp"

using namespace ark_circom;

static uint64_t fnv(const void* p, size_t n, uint64_t h = 1469598103934665603ULL) {
    const uint8_t* b = (const uint8_t*)p;
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ULL; }
    return h;
}

// a decimal scalar below 2^256
static BigInt256 parse_dec(const std::string& s) {
    BigInt256 b = {{0, 0, 0, 0}};
    if (s.empty()) throw std::invalid_argument("empty scalar");
    for (char c : s) {
        if (c < '0' || c > '9') throw std::invalid_argument("not a decimal scalar: " + s);
        unsigned __int128 carry = (unsigned)(c - '0');
        for (int i = 0; i < 4; i++) {
            const unsigned __int128 t = (unsigned __int128)b.l[i] * 10 + carry;
            b.l[i] = (uint64_t)t;
            carry = t >> 64;
        }
        if (carry) throw std::invalid_argument("scalar too long: " + s);
    }
    return b;
}

// r - (v mod r), and 0 for a multiple of r: how snarkjs maps a negative input
static BigInt256 negate_mod_r(BigInt256 v) {
    auto sub = [](BigInt256& x, const uint64_t* y) {
        unsigned __int128 br = 0;
        for (int j = 0; j < 4; j++) { const unsigned __int128 t = (unsigned __int128)x.l[j] - y[j] - br; x.l[j] = (uint64_t)t; br = (t >> 64) & 1; }
    };
    while (ark_circom::detail::geq(v.l, ark_circom::detail::FR_P)) sub(v, ark_circom::detail::FR_P);
    if (!(v.l[0] | v.l[1] | v.l[2] | v.l[3])) return v;
    BigInt256 r; memcpy(r.l, ark_circom::detail::FR_P, 32);
    sub(r, v.l);
    return r;
}

static BigInt256 parse_hex(const std::string& s) {
    BigInt256 b = {{0, 0, 0, 0}};
    std::string t = s.rfind("0x", 0) == 0 ? s.substr(2) : s;
    if (t.size() > 64) throw std::invalid_argument("scalar too long");
    for (char c : t) {
        int v = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : (c >= 'A' && c <= 'F') ? c - 'A' + 10 : -1;
        if (v < 0) throw std::invalid_argument("bad hex digit");
        for (int i = 3; i > 0; i--) b.l[i] = (b.l[i] << 4) | (b.l[i - 1] >> 60);
        b.l[0] = (b.l[0] << 4) | (uint64_t)v;
    }
    return b;
}

// witness of the squaring chain [1, c, a, a^2, a^4, ...] (App. B.4 of SURVEY.md), Montgomery form
static std::vector<Fr> chain_witness(size_t n_vars, uint64_t a) {
    std::vector<Fr> w(n_vars);
    w[0] = Fr::from_u64(1);
    if (n_vars > 2) w[2] = Fr::from_u64(a);
    for (size_t k = 3; k < n_vars; k++) detail::fr_mont_mul(w[k].l, w[k - 1].l, w[k - 1].l);
    if (n_vars > 2) detail::fr_mont_mul(w[1].l, w[n_vars - 1].l, w[n_vars - 1].l);
    return w;
}

int main(int argc, char** argv) {
    try {
        if (argc >= 3 && std::string(argv[1]) == "--parse-only") {
            std::ifstream f(argv[2], std::ios::binary);
            if (!f) throw SerializationError("cannot open zkey");
            auto kv = read_zkey(f);
            const ProvingKey& pk = kv.first; const ConstraintMatrices& m = kv.second;
            std::printf("n_vars=%zu n_public=%zu domain=%zu num_constraints=%zu num_instance=%zu num_witness=%zu a_nnz=%zu b_nnz=%zu\n",
                        pk.a_query.size(), pk.vk.gamma_abc_g1.size() - 1, pk.h_query.size(), m.num_constraints, m.num_instance_variables,
                        m.num_witness_variables, m.a_num_non_zero, m.b_num_non_zero);
            std::printf("fnv a=%016llx b1=%016llx b2=%016llx l=%016llx h=%016llx alpha=%016llx\n",
                        (unsigned long long)fnv(pk.a_query.data(), pk.a_query.size() * 64), (unsigned long long)fnv(pk.b_g1_query.data(), pk.b_g1_query.size() * 64),
                        (unsigned long long)fnv(pk.b_g2_query.data(), pk.b_g2_query.size() * 128), (unsigned long long)fnv(pk.l_query.data(), pk.l_query.size() * 64),
                        (unsigned long long)fnv(pk.h_query.data(), pk.h_query.size() * 64), (unsigned long long)fnv(&pk.vk.alpha_g1, 64));
            uint64_t hc = 1469598103934665603ULL;
            for (const Matrix* mm : {&m.a, &m.b})
                for (const auto& row : *mm) for (const auto& e : row) { hc = fnv(e.first.l, 32, hc); uint32_t c = (uint32_t)e.second; hc = fnv(&c, 4, hc); }
            std::printf("fnv coefs=%016llx\n", (unsigned long long)hc);
            if (argc >= 4 && std::string(argv[3]) == "--dump-key") {       // every query point as the zkey's own bytes (small keys)
                auto dump = [](const char* name, const void* p, size_t count, size_t stride) {
                    const uint8_t* b = (const uint8_t*)p;
                    for (size_t i = 0; i < count; i++) {
                        std::printf("%s[%zu]=", name, i);
                        for (size_t k = 0; k < stride; k++) std::printf("%02x", b[i * stride + k]);
                        std::printf("\n");
                    }
                };
                dump("gamma_abc_g1", pk.vk.gamma_abc_g1.data(), pk.vk.gamma_abc_g1.size(), 64);
                dump("a_query", pk.a_query.data(), pk.a_query.size(), 64);
                dump("b_g1_query", pk.b_g1_query.data(), pk.b_g1_query.size(), 64);
                dump("b_g2_query", pk.b_g2_query.data(), pk.b_g2_query.size(), 128);
                dump("l_query", pk.l_query.data(), pk.l_query.size(), 64);
                dump("h_query", pk.h_query.data(), pk.h_query.size(), 64);
            }
            return 0;
        }
        if (argc >= 4 && std::string(argv[1]) == "--verify") {              // host-only: --verify <zkey> <proof_hex> [public inputs, decimal u64 or 0x hex]
            std::ifstream f(argv[2], std::ios::binary);
            if (!f) throw SerializationError("cannot open zkey");
            auto kv = read_zkey(f);
            std::string hx = argv[3];
            if (hx.size() != 512) throw std::invalid_argument("proof must be 256 bytes of hex");
            Proof proof;
            for (int i = 0; i < 256; i++) proof.bytes[i] = (uint8_t)std::stoul(hx.substr(2 * i, 2), nullptr, 16);
            std::vector<Fr> inputs;
            for (int i = 4; i < argc; i++) { std::string a = argv[i]; inputs.push_back(a.rfind("0x", 0) == 0 ? Fr::from_bigint(parse_hex(a)) : Fr::from_u64(std::stoull(a))); }
            auto pvk = Groth16::process_vk(kv.first.vk);                    // src/zkey.rs:868
            std::printf("verified=%d\n", Groth16::verify_with_processed_vk(pvk, inputs, proof) ? 1 : 0);
            return 0;
        }
        if (argc >= 4 && std::string(argv[1]) == "--ethereum") {            // host-only: the Ethereum views (src/ethereum.rs) and their way back
            namespace eth = ark_circom::ethereum;
            std::ifstream f(argv[2], std::ios::binary);
            if (!f) throw SerializationError("cannot open zkey");
            auto kv = read_zkey(f);
            std::string hx = argv[3];
            if (hx.size() != 512) throw std::invalid_argument("proof must be 256 bytes of hex");
            Proof proof;
            for (int i = 0; i < 256; i++) proof.bytes[i] = (uint8_t)std::stoul(hx.substr(2 * i, 2), nullptr, 16);
            std::vector<Fr> inputs;
            for (int i = 4; i < argc; i++) { std::string a = argv[i]; inputs.push_back(a.rfind("0x", 0) == 0 ? Fr::from_bigint(parse_hex(a)) : Fr::from_u64(std::stoull(a))); }
            const eth::VerifyingKey evk = eth::VerifyingKey::from(kv.first.vk);
            const eth::Proof ep = eth::Proof::from(proof);
            auto g1s = [](const eth::G1& g) { auto t = g.as_tuple(); return t[0].hex() + "," + t[1].hex(); };
            auto g2s = [](const eth::G2& g) { auto t = g.as_tuple(); return t[0][0].hex() + "," + t[0][1].hex() + "," + t[1][0].hex() + "," + t[1][1].hex(); };
            std::printf("vk.alpha1=%s\nvk.beta2=%s\nvk.gamma2=%s\nvk.delta2=%s\n", g1s(evk.alpha1).c_str(), g2s(evk.beta2).c_str(), g2s(evk.gamma2).c_str(), g2s(evk.delta2).c_str());
            for (size_t i = 0; i < evk.ic.size(); i++) std::printf("vk.ic[%zu]=%s\n", i, g1s(evk.ic[i]).c_str());
            std::printf("proof.a=%s\nproof.b=%s\nproof.c=%s\ncalldata=", g1s(ep.a).c_str(), g2s(ep.b).c_str(), g1s(ep.c).c_str());
            for (const eth::U256& w : ep.calldata_words()) std::printf("%s", w.hex().c_str());
            std::printf("\n");
            const std::vector<eth::U256> ein = eth::inputs(inputs);
            for (size_t i = 0; i < ein.size(); i++) std::printf("inputs[%zu]=%s\n", i, ein[i].hex().c_str());
            // the reference's convert_vk / convert_proof / convert_fr tests (src/ethereum.rs:195-279), then check_proof with the host verifier
            const VerifyingKey vk2 = evk.into();
            bool rt = !memcmp(&vk2.alpha_g1, &kv.first.vk.alpha_g1, 64) && !memcmp(&vk2.beta_g2, &kv.first.vk.beta_g2, 128) &&
                      !memcmp(&vk2.gamma_g2, &kv.first.vk.gamma_g2, 128) && !memcmp(&vk2.delta_g2, &kv.first.vk.delta_g2, 128) &&
                      vk2.gamma_abc_g1.size() == kv.first.vk.gamma_abc_g1.size();
            for (size_t i = 0; rt && i < vk2.gamma_abc_g1.size(); i++) rt = !memcmp(&vk2.gamma_abc_g1[i], &kv.first.vk.gamma_abc_g1[i], 64);
            const Proof p2 = ep.into();
            rt = rt && !memcmp(p2.bytes, proof.bytes, 256) && eth::Proof::from(p2) == ep;
            std::vector<Fr> in2;
            for (const eth::U256& w : ein) in2.push_back(eth::u256_to_fr(w));
            for (size_t i = 0; i < inputs.size(); i++) rt = rt && in2[i] == inputs[i];
            std::printf("roundtrip=%d\ncompressed=", rt ? 1 : 0);            // Proof::serialize_compressed
            for (uint8_t b : serialize_compressed(proof)) std::printf("%02x", b);
            std::printf("\n");
            std::printf("verified=%d\n", Groth16::verify_with_processed_vk(Groth16::process_vk(vk2), in2, p2) ? 1 : 0);
            return 0;
        }
        if (const char* ptau = std::getenv("B2G_PTAU_PREPARE")) {           // ceremony -> its Lagrange sections -> a prepared file
            if (argc < 2) { std::fprintf(stderr, "usage: B2G_PTAU_PREPARE=<in.ptau> %s <out.ptau> [power]\n", argv[0]); return 2; }
            const uint32_t power = argc > 2 ? (uint32_t)std::stoul(argv[2]) : 0;
            std::ifstream pf(ptau, std::ios::binary);
            if (!pf) throw SerializationError("cannot open ptau");
            const Powers powers = read_ptau(pf, power);
            typedef Groth16T<CircomReduction> G;
            const auto t0 = std::chrono::steady_clock::now();
            const Powers prepared = G::prepare_powers_of_tau(powers, power);
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            std::ofstream of(argv[1], std::ios::binary);
            if (!of) throw SerializationError("cannot open the output file");
            write_ptau(of, prepared);
            std::printf("power=%u\nms=%.3f\n", prepared.power, ms);
            return 0;
        }
        if (const char* ptau = std::getenv("B2G_PTAU_CONTRIBUTE")) {        // ceremony -> one contribution -> a new file
            if (argc != 2 && argc != 5) {
                std::fprintf(stderr, "usage: B2G_PTAU_CONTRIBUTE=<in.ptau> %s <out.ptau> [tau alpha beta]\n", argv[0]);
                return 2;
            }
            std::ifstream pf(ptau, std::ios::binary);
            if (!pf) throw SerializationError("cannot open ptau");
            const Powers powers = read_ptau(pf);
            typedef Groth16T<CircomReduction> G;
            const auto t0 = std::chrono::steady_clock::now();
            Powers out;
            if (argc == 5) {
                BigInt256 s[3];
                for (int k = 0; k < 3; k++) s[k] = parse_dec(argv[2 + k]);
                out = G::contribute_powers_of_tau(powers, s[0], s[1], s[2]);
            } else {
                out = G::contribute_powers_of_tau(powers);
            }
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            std::ofstream of(argv[1], std::ios::binary);
            if (!of) throw SerializationError("cannot open the output file");
            write_ptau(of, out);
            std::printf("power=%u\nms=%.3f\n", out.power, ms);
            return 0;
        }
        if (const char* ptau = std::getenv("B2G_PTAU_CHECK")) {             // ceremony -> its check on the GPU
            const uint32_t log_n = argc > 1 ? (uint32_t)std::stoul(argv[1]) : 0;
            std::ifstream pf(ptau, std::ios::binary);
            if (!pf) throw SerializationError("cannot open ptau");
            const Powers powers = read_ptau(pf, log_n);
            typedef Groth16T<CircomReduction> G;
            const auto t0 = std::chrono::steady_clock::now();
            const PowersCheck r = G::verify_powers_of_tau(powers, log_n);
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            std::printf("powers=%d\n", r.ok ? 1 : 0);
            if (!r.ok) std::printf("reason=%s\n", r.reason().c_str());
            std::printf("ms=%.3f\n", ms);
            return 0;
        }
        if (const char* ptau = std::getenv("B2G_ZKEY_VERIFY")) {            // R1CS + ceremony + zkey -> the key's check on the GPU
            if (argc < 3) { std::fprintf(stderr, "usage: B2G_ZKEY_VERIFY=<file.ptau> %s <circuit.r1cs> <circuit.zkey>\n", argv[0]); return 2; }
            std::ifstream rf(argv[1], std::ios::binary);
            if (!rf) throw SerializationError("cannot open r1cs");
            const ConstraintMatrices matrices = R1CS::read(rf).to_matrices();
            std::ifstream zf(argv[2], std::ios::binary);
            if (!zf) throw SerializationError("cannot open zkey");
            const auto key = read_zkey(zf);
            uint32_t log_n = 1;
            while ((1ull << log_n) < matrices.num_constraints + matrices.num_instance_variables) log_n++;
            std::ifstream pf(ptau, std::ios::binary);
            if (!pf) throw SerializationError("cannot open ptau");
            const Powers powers = read_ptau(pf, log_n);
            typedef Groth16T<CircomReduction> G;
            const auto t0 = std::chrono::steady_clock::now();
            const SetupCheck r = G::verify_proving_key(matrices, powers, key.first, &key.second);
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            std::printf("key=%d", r.ok ? 1 : 0);
            if (!r.ok) std::printf(" %s", r.reason().c_str());
            std::printf("\nms=%.3f\n", ms);
            return 0;
        }
        if (const char* ptau = std::getenv("B2G_SETUP_PTAU")) {             // R1CS + ceremony -> key -> contribution -> check -> prove -> verify
            if (argc < 3) { std::fprintf(stderr, "usage: B2G_SETUP_PTAU=<file.ptau> %s <circuit.r1cs> <witness.wtns> [seed]\n", argv[0]); return 2; }
            typedef Groth16T<CircomReduction> G;
            std::ifstream rf(argv[1], std::ios::binary);
            if (!rf) throw SerializationError("cannot open r1cs");
            const ConstraintMatrices matrices = R1CS::read(rf).to_matrices();
            std::ifstream wf(argv[2], std::ios::binary);
            if (!wf) throw SerializationError("cannot open wtns");
            const std::vector<Fr> w = read_wtns(wf);
            uint32_t log_n = 0;
            while ((1ull << log_n) < matrices.num_constraints + matrices.num_instance_variables) log_n++;
            std::ifstream pf(ptau, std::ios::binary);
            if (!pf) throw SerializationError("cannot open ptau");
            const Powers powers = read_ptau(pf, log_n ? log_n : 1);
            const ProvingKey pk0 = G::generate_parameters_from_powers_of_tau(matrices, powers);
            std::mt19937_64 rng(std::stoull(argc > 3 ? argv[3] : "0x5E7", nullptr, 0));
            std::mt19937_64 replay = rng;                                    // the same draw, to print x
            Fr x;
            while (x.is_zero()) x = Fr::rand(replay);
            const BigInt256 xb = x.into_bigint();
            std::printf("x=0x%016llx%016llx%016llx%016llx\n", (unsigned long long)xb.l[3], (unsigned long long)xb.l[2],
                        (unsigned long long)xb.l[1], (unsigned long long)xb.l[0]);
            const ProvingKey pk = G::contribute(pk0, rng);
            std::printf("key=");
            for (uint8_t b : serialize_proving_key(pk)) std::printf("%02x", b);
            std::printf("\ncontribution=%d\n", G::verify_contribution(pk0, pk) ? 1 : 0);
            const Proof proof = G::prove(pk, matrices, w, rng);
            std::printf("proof=%s\n", proof.hex().c_str());
            const std::vector<Fr> inputs(w.begin() + 1, w.begin() + matrices.num_instance_variables);
            std::printf("verified=%d\n", G::verify_with_processed_vk(G::process_vk(pk.vk), inputs, proof) ? 1 : 0);
            return 0;
        }
        if (const char* wasm = std::getenv("B2G_WITNESS")) {                // .wasm + inputs -> witnesses on the GPU -> setup -> prove -> verify
            if (argc < 3) { std::fprintf(stderr, "usage: B2G_WITNESS=<circuit.wasm> %s <circuit.r1cs> name=value ... [count]\n", argv[0]); return 2; }
            typedef Groth16T<LibsnarkReduction> G;
            std::ifstream rf(argv[1], std::ios::binary);
            if (!rf) throw SerializationError("cannot open r1cs");
            const R1CS r1cs = R1CS::read(rf);
            const ConstraintMatrices matrices = r1cs.to_matrices();
            WitnessCalculator::Inputs inputs;
            size_t count = 1;
            for (int i = 2; i < argc; i++) {                                 // name=value (decimal, a leading - maps to r - |v|), repeated for arrays
                const std::string a = argv[i];
                const size_t eq = a.find('=');
                if (eq == std::string::npos) { count = std::stoul(a); continue; }
                const std::string name = a.substr(0, eq), val = a.substr(eq + 1);
                const bool neg = !val.empty() && val[0] == '-';
                BigInt256 v = parse_dec(neg ? val.substr(1) : val);
                if (neg) v = negate_mod_r(v);
                auto it = std::find_if(inputs.begin(), inputs.end(), [&](const auto& e) { return e.first == name; });
                if (it == inputs.end()) inputs.push_back({name, {v}}); else it->second.push_back(v);
            }
            WitnessCalculator calc = WitnessCalculator::from_file(wasm);
            std::vector<std::vector<Fr>> ws; std::vector<uint32_t> status;
            const auto t0 = std::chrono::steady_clock::now();
            calc.calculate_witnesses(std::vector<WitnessCalculator::Inputs>(count, inputs), ws, status);
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            for (size_t i = 0; i < count; i++)
                if (status[i]) { std::printf("witness %zu: %s\n", i, WitnessCalculator::status_name(status[i])); return 1; }
            std::printf("witnesses %zu x %u wires in %.3f ms (%.1f witnesses/s, including the module's device state set-up)\n",
                        count, calc.witness_size, ms, count / (ms * 1e-3));
            if (const char* out = std::getenv("B2G_WITNESS_OUT")) {          // the Montgomery witnesses, witness-major
                std::ofstream of(out, std::ios::binary);
                for (const auto& w : ws) of.write((const char*)w.data(), w.size() * sizeof(Fr));
            }
            std::mt19937_64 rng(0x5EED);
            const ProvingKey pk = G::generate_random_parameters_with_reduction(matrices, rng);
            std::vector<std::pair<Fr, Fr>> rs;
            std::vector<const std::vector<Fr>*> ptrs;
            std::vector<std::vector<Fr>> pubs;
            for (size_t i = 0; i < count; i++) {
                const Fr r = Fr::rand(rng), s2 = Fr::rand(rng);
                rs.push_back({r, s2});
                ptrs.push_back(&ws[i]);
                pubs.emplace_back(ws[i].begin() + 1, ws[i].begin() + matrices.num_instance_variables);
            }
            const std::vector<Proof> proofs = G::create_proofs(pk, matrices, rs, ptrs);
            const std::vector<bool> ok = G::verify_many(G::process_vk(pk.vk), pubs, proofs);
            const size_t good = (size_t)std::count(ok.begin(), ok.end(), true);
            std::printf("verified %zu/%zu\n", good, count);
            return good == count ? 0 : 1;
        }
        if (const char* seed = std::getenv("B2G_SETUP")) {                  // R1CS -> setup on the GPU -> prove -> verify
            if (argc < 3) { std::fprintf(stderr, "usage: B2G_SETUP=<seed> %s <circuit.r1cs> <witness.wtns>\n", argv[0]); return 2; }
            typedef Groth16T<LibsnarkReduction> G;                           // Groth16<Bn254> (tests/groth16.rs:9)
            std::ifstream rf(argv[1], std::ios::binary);
            if (!rf) throw SerializationError("cannot open r1cs");
            const R1CS r1cs = R1CS::read(rf);
            const ConstraintMatrices matrices = r1cs.to_matrices();
            std::ifstream wf(argv[2], std::ios::binary);
            if (!wf) throw SerializationError("cannot open wtns");
            const std::vector<Fr> w = read_wtns(wf);
            std::mt19937_64 rng(std::stoull(seed, nullptr, 0));
            std::mt19937_64 replay = rng;                                    // the same draws, to print the secrets
            const char* names[5] = {"alpha", "beta", "gamma", "delta", "tau"};
            for (const char* name : names) {
                const BigInt256 b = Fr::rand(replay).into_bigint();
                std::printf("%s=0x%016llx%016llx%016llx%016llx\n", name, (unsigned long long)b.l[3], (unsigned long long)b.l[2],
                            (unsigned long long)b.l[1], (unsigned long long)b.l[0]);
            }
            const ProvingKey pk = G::generate_random_parameters_with_reduction(matrices, rng);
            std::printf("key=");
            for (uint8_t b : serialize_proving_key(pk)) std::printf("%02x", b);
            std::printf("\n");
            const Proof proof = G::prove(pk, matrices, w, rng);
            std::printf("proof=%s\n", proof.hex().c_str());
            const std::vector<Fr> inputs(w.begin() + 1, w.begin() + matrices.num_instance_variables);
            std::printf("verified=%d\n", G::verify_with_processed_vk(G::process_vk(pk.vk), inputs, proof) ? 1 : 0);
            return 0;
        }
        if (argc < 3) { std::fprintf(stderr, "usage: %s [--parse-only] <zkey> chain:<a>|<wtns> [iters] [r_hex s_hex]\n", argv[0]); return 2; }
        std::ifstream f(argv[1], std::ios::binary);
        if (!f) throw SerializationError("cannot open zkey");
        auto kv = read_zkey(f);                                     // benches/groth16.rs:20-23
        const ProvingKey& params = kv.first; const ConstraintMatrices& matrices = kv.second;
        const size_t num_inputs = matrices.num_instance_variables, num_constraints = matrices.num_constraints;
        std::string wsrc = argv[2];
        std::vector<Fr> full_assignment;
        if (wsrc.rfind("chain:", 0) == 0) full_assignment = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)));
        else { std::ifstream wf(wsrc, std::ios::binary); if (!wf) throw SerializationError("cannot open wtns"); full_assignment = read_wtns(wf); }
        int iters = argc > 3 ? std::atoi(argv[3]) : 10;
        Fr r, s;
        if (argc > 5) { r = Fr::from_bigint(parse_hex(argv[4])); s = Fr::from_bigint(parse_hex(argv[5])); }
        else { std::mt19937_64 rng(0xB200); r = Fr::rand(rng); s = Fr::rand(rng); }      // benches/groth16.rs:45-50
        Proof proof = Groth16::create_proof_with_reduction_and_matrices(params, r, s, matrices, num_inputs, num_constraints, full_assignment);
        std::printf("proof=%s\n", proof.hex().c_str());
        {   // src/zkey.rs:868-872: process_vk, public inputs = w[1..num_inputs] (circuit.rs:18-26), verify_with_processed_vk
            auto pvk = Groth16::process_vk(params.vk);
            std::vector<Fr> inputs(full_assignment.begin() + 1, full_assignment.begin() + num_inputs);
            std::printf("verified=%d\n", Groth16::verify_with_processed_vk(pvk, inputs, proof) ? 1 : 0);
        }
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; i++)                             // benches/groth16.rs:69-84
            proof = Groth16::create_proof_with_reduction_and_matrices(params, r, s, matrices, num_inputs, num_constraints, full_assignment);
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / (iters > 0 ? iters : 1);
        std::printf("groth proof %zu constraints: %.3f ms/proof over %d iterations\n", num_constraints, ms, iters);
        if (const char* inf = std::getenv("B2G_INFLIGHT")) {              // pipelined: one host thread, several proofs queued on the GPU
            const int k = std::atoi(inf), total = iters > 0 ? 3 * iters : 3;
            std::vector<std::pair<Fr, Fr>> rs((size_t)total, {r, s});
            std::vector<const std::vector<Fr>*> ws((size_t)total, &full_assignment);
            Groth16::prove_batch(params, matrices, {rs[0]}, {ws[0]}, 1);                        // warm-up: loads the key on a fresh context
            auto t1 = std::chrono::steady_clock::now();
            std::vector<Proof> proofs = Groth16::prove_batch(params, matrices, rs, ws, k);
            double pms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count() / total;
            bool same = true;
            for (const Proof& q : proofs) same = same && !memcmp(q.bytes, proof.bytes, 256);
            std::printf("pipelined (%d in flight, one host thread, includes key load on %d contexts): %.3f ms/proof over %d proofs, identical=%d\n", k, k, pms, total, same ? 1 : 0);
        }
        if (const char* many = std::getenv("B2G_MANY")) {                 // batched: K proofs in one device pass (Groth16::create_proofs)
            const int k = std::atoi(many);
            if (k < 1) throw SynthesisError("B2G_MANY must be >= 1");
            // proof i proves chain:<a + i> (or the .wtns for every i) with the same (r, s); proof 0 is the one printed above
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::vector<std::pair<Fr, Fr>> rs((size_t)k, {r, s});
            std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);   // also the warm-up of this count
            const int reps = iters > 0 ? iters : 1;
            auto t1 = std::chrono::steady_clock::now();
            for (int it = 0; it < reps; it++) proofs = Groth16::create_proofs(params, matrices, rs, ws);
            double pms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count() / ((double)reps * k);
            for (int i = 0; i < k; i++) std::printf("many[%d]=%s\n", i, proofs[(size_t)i].hex().c_str());
            std::printf("batched (%d proofs in one device pass, one context): %.3f ms/proof over %d calls, first_identical=%d\n", k, pms, reps,
                        !memcmp(proofs[0].bytes, proof.bytes, 256) ? 1 : 0);
        }
        if (const char* pkeys = std::getenv("B2G_PROVE_KEYS")) {          // K copies of the key, one proof each, in one device pass
            const int k = std::atoi(pkeys);
            if (k < 1) throw SynthesisError("B2G_PROVE_KEYS must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<std::pair<const ProvingKey*, const ConstraintMatrices*>> keys((size_t)k, {&params, &matrices});
            auto group = Groth16::load_proving_keys(keys);
            std::vector<Groth16::KeyBatch> batches;
            for (int i = 0; i < k; i++) batches.push_back({{{r, s}}, {&wv[(size_t)i]}});
            auto proofs = Groth16::create_proofs_keys(*group, batches);      // also the warm-up of this shape
            const int reps = iters > 0 ? iters : 1;
            auto t1 = std::chrono::steady_clock::now();
            for (int it = 0; it < reps; it++) proofs = Groth16::create_proofs_keys(*group, batches);
            double pms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count() / ((double)reps * k);
            for (int i = 0; i < k; i++) std::printf("keys[%d]=%s\n", i, proofs[(size_t)i][0].hex().c_str());
            std::printf("keyed (%d keys, one proof each, in one device pass): %.3f ms/proof over %d calls, first_identical=%d\n", k, pms, reps,
                        !memcmp(proofs[0][0].bytes, proof.bytes, 256) ? 1 : 0);
        }
        if (const char* vm = std::getenv("B2G_VERIFY_MANY")) {           // batched verification against the host verifier
            const int k = std::atoi(vm);
            if (k < 1) throw SynthesisError("B2G_VERIFY_MANY must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0xC0DE);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            std::vector<std::vector<Fr>> inputs;
            for (const auto& w : wv) inputs.emplace_back(w.begin() + 1, w.begin() + num_inputs);
            for (int i = 1; i < k; i += 2) {                              // A -> -A: y -> p - y (y != 0 on the curve)
                uint64_t y[4], d[4]; memcpy(y, proofs[(size_t)i].bytes + 32, 32);
                unsigned __int128 borrow = 0;
                for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
                memcpy(proofs[(size_t)i].bytes + 32, d, 32);
            }
            auto pvk = Groth16::process_vk(params.vk);
            std::vector<bool> got = Groth16::verify_many(pvk, inputs, proofs);    // also loads the key on the device
            auto t1 = std::chrono::steady_clock::now();
            got = Groth16::verify_many(pvk, inputs, proofs);
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            int agree = 1, valid = 0;
            auto t2 = std::chrono::steady_clock::now();
            for (int i = 0; i < k; i++) {
                const bool host = Groth16::verify_with_processed_vk(pvk, inputs[(size_t)i], proofs[(size_t)i]);
                agree &= host == got[(size_t)i];
                valid += host;
            }
            const double host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t2).count();
            std::printf("verify_many %d proofs (%d valid): agree=%d, device %.3f ms/batch (%.1f proofs/s), host verify_with_processed_vk "
                        "%.3f ms/proof on one core (%.1f proofs/s)\n", k, valid, agree, dev_ms, k / (dev_ms / 1e3), host_ms / k, k / (host_ms / 1e3));
        }
        if (const char* vb = std::getenv("B2G_VERIFY_BATCH")) {          // one batch verdict against the host verifier
            const int k = std::atoi(vb);
            if (k < 1) throw SynthesisError("B2G_VERIFY_BATCH must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0xBA7C);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            std::vector<std::vector<Fr>> inputs;
            for (const auto& w : wv) inputs.emplace_back(w.begin() + 1, w.begin() + num_inputs);
            auto pvk = Groth16::process_vk(params.vk);
            const bool valid = Groth16::verify_batch(pvk, inputs, proofs);      // also loads the key on the device
            auto t1 = std::chrono::steady_clock::now();
            const bool again = Groth16::verify_batch(pvk, inputs, proofs);
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            std::vector<Proof> bad = proofs;                                 // the last proof's A -> -A: y -> p - y
            uint64_t y[4], d[4]; memcpy(y, bad.back().bytes + 32, 32);
            unsigned __int128 borrow = 0;
            for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
            memcpy(bad.back().bytes + 32, d, 32);
            const bool tampered = Groth16::verify_batch(pvk, inputs, bad);
            bool host = true, host_bad = true;
            for (int i = 0; i < k; i++) {
                host = host && Groth16::verify_with_processed_vk(pvk, inputs[(size_t)i], proofs[(size_t)i]);
                host_bad = host_bad && Groth16::verify_with_processed_vk(pvk, inputs[(size_t)i], bad[(size_t)i]);
            }
            std::printf("verify_batch %d proofs: valid=%d tampered=%d host=%d/%d agree=%d, device %.3f ms/batch (%.1f proofs/s)\n", k,
                        valid && again, tampered, host, host_bad, (valid && again) == host && tampered == host_bad, dev_ms, k / (dev_ms / 1e3));
        }
        if (const char* vc = std::getenv("B2G_VERIFY_COMPRESSED")) {     // compressed proofs decoded on the device, against the host
            const int k = std::atoi(vc);
            if (k < 1) throw SynthesisError("B2G_VERIFY_COMPRESSED must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0xC0C0);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            const std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            std::vector<std::vector<Fr>> inputs;
            for (const auto& w : wv) inputs.emplace_back(w.begin() + 1, w.begin() + num_inputs);
            std::vector<CompressedProof> blobs, flipped;
            for (const Proof& p : proofs) blobs.push_back(serialize_compressed(p));
            flipped = blobs;
            for (int i = 1; i < k; i += 2) flipped[(size_t)i][31] ^= 0x80;  // the sign bit of A: A -> -A
            std::vector<Proof> negated = proofs;                          // the same proofs uncompressed: y -> p - y
            for (int i = 1; i < k; i += 2) {
                uint64_t y[4], d[4]; memcpy(y, negated[(size_t)i].bytes + 32, 32);
                unsigned __int128 borrow = 0;
                for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
                memcpy(negated[(size_t)i].bytes + 32, d, 32);
            }
            auto pvk = Groth16::process_vk(params.vk);
            const std::vector<bool> got = Groth16::verify_many_compressed(pvk, inputs, flipped);
            int agree = 1, valid = 0;
            for (int i = 0; i < k; i++) {
                const bool host = Groth16::verify_with_processed_vk(pvk, inputs[(size_t)i], negated[(size_t)i]);
                agree &= host == got[(size_t)i];
                valid += host;
            }
            const auto decoded = Groth16::decompress_proofs(blobs);
            int round_trip = 1;
            for (int i = 0; i < k; i++) round_trip &= decoded[(size_t)i].has_value() && !memcmp(decoded[(size_t)i]->bytes, proofs[(size_t)i].bytes, 256);
            const bool batch = Groth16::verify_batch_compressed(pvk, inputs, blobs), batch_flipped = Groth16::verify_batch_compressed(pvk, inputs, flipped);
            std::printf("verify_compressed %d proofs (%d valid): many agree=%d, batch valid=%d flipped=%d, round trip=%d\n", k, valid, agree,
                        batch, batch_flipped, round_trip);
        }
        if (const char* vl = std::getenv("B2G_VERIFY_LOCATE")) {         // per-proof verdicts of the grouped batch check, against the host
            const int k = std::atoi(vl);
            if (k < 1) throw SynthesisError("B2G_VERIFY_LOCATE must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0x10CA);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            std::vector<std::vector<Fr>> inputs;
            for (const auto& w : wv) inputs.emplace_back(w.begin() + 1, w.begin() + num_inputs);
            std::vector<size_t> at = {0, (size_t)k / 2, (size_t)k - 1};
            std::sort(at.begin(), at.end());
            at.erase(std::unique(at.begin(), at.end()), at.end());
            for (size_t i : at) {                                         // A -> -A: y -> p - y
                uint64_t y[4], d[4]; memcpy(y, proofs[i].bytes + 32, 32);
                unsigned __int128 borrow = 0;
                for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
                memcpy(proofs[i].bytes + 32, d, 32);
            }
            auto pvk = Groth16::process_vk(params.vk);
            std::vector<bool> got = Groth16::verify_batch_locate(pvk, inputs, proofs);   // also loads the key on the device
            auto t1 = std::chrono::steady_clock::now();
            got = Groth16::verify_batch_locate(pvk, inputs, proofs);
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            int agree = 1, valid = 0;
            for (int i = 0; i < k; i++) {
                const bool host = Groth16::verify_with_processed_vk(pvk, inputs[(size_t)i], proofs[(size_t)i]);
                agree &= host == got[(size_t)i];
                valid += host;
            }
            std::printf("verify_locate %d proofs (%d valid, %d tampered): agree=%d, device %.3f ms/batch (%.1f proofs/s)\n", k, valid,
                        (int)at.size(), agree, dev_ms, k / (dev_ms / 1e3));
        }
        if (const char* vk_env = std::getenv("B2G_VERIFY_KEYS")) {       // one verdict per key batch, against the host
            const int k = std::atoi(vk_env);
            if (k < 1) throw SynthesisError("B2G_VERIFY_KEYS must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0x4E75);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            const std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            // the proofs split into up to four batches of the bench key (sizes about k/4, the rest in the last), plus an empty
            // one; the last proof of the second batch (or of the first, with one batch) gets A -> -A
            const size_t nb = std::min<size_t>(4, (size_t)k), per = (size_t)k / nb;
            std::vector<std::vector<std::vector<Fr>>> inputs(nb + 1);
            std::vector<std::vector<Proof>> parts(nb + 1);
            for (size_t i = 0; i < (size_t)k; i++) {
                const size_t b = std::min(i / per, nb - 1);
                inputs[b].emplace_back(wv[i].begin() + 1, wv[i].begin() + num_inputs);
                parts[b].push_back(proofs[i]);
            }
            Proof& bad = parts[nb > 1 ? 1 : 0].back();
            uint64_t y[4], d[4]; memcpy(y, bad.bytes + 32, 32);
            unsigned __int128 borrow = 0;
            for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
            memcpy(bad.bytes + 32, d, 32);
            auto pvk = Groth16::process_vk(params.vk);
            std::vector<KeyBatch> batches;
            for (size_t b = 0; b <= nb; b++) batches.push_back({pvk, inputs[b], parts[b]});
            std::vector<bool> got = Groth16::verify_batch_keys(batches);        // also loads the key on the device
            auto t1 = std::chrono::steady_clock::now();
            got = Groth16::verify_batch_keys(batches);
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            std::string dev, host;
            for (size_t b = 0; b <= nb; b++) {
                bool h = true;
                for (size_t i = 0; i < parts[b].size(); i++) h = h && Groth16::verify_with_processed_vk(pvk, inputs[b][i], parts[b][i]);
                dev += got[b] ? '1' : '0';
                host += h ? '1' : '0';
            }
            std::printf("verify_keys %d proofs in %d batches: device=%s host=%s agree=%d, device %.3f ms/call (%.1f proofs/s)\n", k,
                        (int)nb + 1, dev.c_str(), host.c_str(), dev == host, dev_ms, k / (dev_ms / 1e3));
        }
        if (const char* lk = std::getenv("B2G_LOAD_KEYS")) {             // K keys prepared in one call, then verified, against the host
            const int k = std::atoi(lk);
            if (k < 1) throw SynthesisError("B2G_LOAD_KEYS must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0x10AD);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            const std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            // k prepared copies of the bench key, each a separate device key; batch i holds proof i under copy i, with A -> -A
            // in every third proof
            const std::vector<PreparedVerifyingKey> pvks((size_t)k, Groth16::process_vk(params.vk));
            std::vector<std::vector<std::vector<Fr>>> inputs((size_t)k);
            std::vector<std::vector<Proof>> parts((size_t)k);
            std::vector<KeyBatch> batches;
            for (size_t i = 0; i < (size_t)k; i++) {
                inputs[i].emplace_back(wv[i].begin() + 1, wv[i].begin() + num_inputs);
                parts[i].push_back(proofs[i]);
                if (i % 3 == 1) {
                    Proof& bad = parts[i].back();
                    uint64_t y[4], d[4]; memcpy(y, bad.bytes + 32, 32);
                    unsigned __int128 borrow = 0;
                    for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
                    memcpy(bad.bytes + 32, d, 32);
                }
            }
            for (size_t i = 0; i < (size_t)k; i++) batches.push_back({pvks[i], inputs[i], parts[i]});
            uint64_t l0 = 0, l1 = 0, l2 = 0;
            check(b2g_launch_count(Gpu::instance().ctx(), &l0));
            auto t1 = std::chrono::steady_clock::now();
            Groth16::load_verifying_keys(pvks);
            const double load_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            check(b2g_launch_count(Gpu::instance().ctx(), &l1));
            bool held = true;
            for (const auto& p : pvks) held = held && p.device.find(Gpu::instance().ctx(), 0);
            const std::vector<bool> got = Groth16::verify_batch_keys(batches);
            check(b2g_launch_count(Gpu::instance().ctx(), &l2));
            std::string dev, host;
            for (size_t i = 0; i < (size_t)k; i++) {
                dev += got[i] ? '1' : '0';
                host += Groth16::verify_with_processed_vk(pvks[i], inputs[i][0], parts[i][0]) ? '1' : '0';
            }
            // the keyed call after load_verifying_keys loads nothing: it issues the launches of a call with preloaded keys
            std::printf("load_keys %d keys: held=%d load_launches=%llu verify_launches=%llu device=%s host=%s agree=%d, load %.3f ms\n", k,
                        held, (unsigned long long)(l1 - l0), (unsigned long long)(l2 - l1), dev.c_str(), host.c_str(), dev == host, load_ms);
        }
        if (const char* kl = std::getenv("B2G_VERIFY_KEYS_LOCATE")) {    // one verdict per proof over key batches, against the host
            const int k = std::atoi(kl);
            if (k < 1) throw SynthesisError("B2G_VERIFY_KEYS_LOCATE must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 rng(0x4C0C);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(rng), Fr::rand(rng)});
            const std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            // up to four batches of the bench key (sizes about k/4, the rest in the last) with an empty one after the first;
            // A -> -A in the first proof of the first batch, the last proof of every other batch, and proofs 63 and 64 (the
            // edge of its first two groups) of every batch that has them
            const size_t nb = std::min<size_t>(4, (size_t)k), per = (size_t)k / nb;
            std::vector<std::vector<std::vector<Fr>>> inputs(nb + 1);
            std::vector<std::vector<Proof>> parts(nb + 1);
            for (size_t i = 0; i < (size_t)k; i++) {
                const size_t b = std::min(i / per, nb - 1);
                const size_t slot = b == 0 ? 0 : b + 1;                    // slot 1 stays empty
                inputs[slot].emplace_back(wv[i].begin() + 1, wv[i].begin() + num_inputs);
                parts[slot].push_back(proofs[i]);
            }
            int tampered = 0;
            for (size_t b = 0; b <= nb; b++) {
                std::vector<size_t> at;
                if (parts[b].empty()) continue;
                at.push_back(b == 0 ? 0 : parts[b].size() - 1);
                if (parts[b].size() > 64) { at.push_back(63); at.push_back(64); }
                std::sort(at.begin(), at.end());
                at.erase(std::unique(at.begin(), at.end()), at.end());
                for (size_t i : at) {                                     // A -> -A: y -> p - y
                    uint64_t y[4], d[4]; memcpy(y, parts[b][i].bytes + 32, 32);
                    unsigned __int128 borrow = 0;
                    for (int j = 0; j < 4; j++) { unsigned __int128 t = (unsigned __int128)detail::FQ_P[j] - y[j] - borrow; d[j] = (uint64_t)t; borrow = (t >> 64) & 1; }
                    memcpy(parts[b][i].bytes + 32, d, 32);
                    tampered++;
                }
            }
            auto pvk = Groth16::process_vk(params.vk);
            std::vector<KeyBatch> batches;
            for (size_t b = 0; b <= nb; b++) batches.push_back({pvk, inputs[b], parts[b]});
            std::vector<std::vector<bool>> got = Groth16::verify_batch_keys_locate(batches);   // also loads the key on the device
            auto t1 = std::chrono::steady_clock::now();
            got = Groth16::verify_batch_keys_locate(batches);
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            int agree = got.size() == nb + 1, valid = 0;
            for (size_t b = 0; b <= nb && agree; b++) {
                agree &= got[b].size() == parts[b].size();
                for (size_t i = 0; i < parts[b].size() && agree; i++) {
                    const bool host = Groth16::verify_with_processed_vk(pvk, inputs[b][i], parts[b][i]);
                    agree &= host == got[b][i];
                    valid += host;
                }
            }
            std::printf("verify_keys_locate %d proofs in %d batches (%d valid, %d tampered): agree=%d, device %.3f ms/call (%.1f proofs/s)\n",
                        k, (int)nb + 1, valid, tampered, agree, dev_ms, k / (dev_ms / 1e3));
        }
        if (const char* rr = std::getenv("B2G_RERANDOMIZE")) {           // rerandomized proofs, rows printed for the Python mirror
            const int k = std::atoi(rr);
            if (k < 1) throw SynthesisError("B2G_RERANDOMIZE must be >= 1");
            std::vector<std::vector<Fr>> wv((size_t)k, full_assignment);
            if (wsrc.rfind("chain:", 0) == 0)
                for (int i = 1; i < k; i++) wv[(size_t)i] = chain_witness(params.a_query.size(), std::stoull(wsrc.substr(6)) + (unsigned long long)i);
            std::vector<const std::vector<Fr>*> ws;
            for (const auto& w : wv) ws.push_back(&w);
            std::mt19937_64 prng(0x4E4D);
            std::vector<std::pair<Fr, Fr>> rs;
            for (int i = 0; i < k; i++) rs.push_back({Fr::rand(prng), Fr::rand(prng)});
            const std::vector<Proof> proofs = Groth16::create_proofs(params, matrices, rs, ws);
            auto pvk = Groth16::process_vk(params.vk);
            std::mt19937_64 rng(0x5EED);
            auto t1 = std::chrono::steady_clock::now();
            const std::vector<std::optional<Proof>> out = Groth16::rerandomize_many(pvk, proofs, rng);   // includes the key load
            const double dev_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            int valid = 0, changed = 0;
            for (int i = 0; i < k; i++) {
                const Proof& q = *out[(size_t)i];
                std::printf("rerand_in[%d]=%s\nrerand[%d]=%s\n", i, proofs[(size_t)i].hex().c_str(), i, q.hex().c_str());
                const std::vector<Fr> inputs(wv[(size_t)i].begin() + 1, wv[(size_t)i].begin() + num_inputs);
                valid += Groth16::verify_with_processed_vk(pvk, inputs, q);
                changed += memcmp(q.bytes, proofs[(size_t)i].bytes, 256) != 0;
            }
            std::printf("rerandomize %d proofs: valid=%d changed=%d, device %.3f ms/call (with the key load)\n", k, valid, changed, dev_ms);
        }
        if (const char* ak = std::getenv("B2G_ARK_KEYS")) {              // the key in both ark-serialize forms, written and read back
            auto same = [](const auto& a, const auto& b) { return a.size() == b.size() && (a.empty() || !memcmp(a.data(), b.data(), a.size() * sizeof(a[0]))); };
            for (int z = 1; z >= 0; z--) {
                const std::string path = std::string(ak) + (z ? ".compressed" : ".uncompressed");
                auto t1 = std::chrono::steady_clock::now();
                const std::vector<uint8_t> bytes = serialize_proving_key(params, z);
                {
                    std::ofstream of(path, std::ios::binary);
                    of.write((const char*)bytes.data(), (std::streamsize)bytes.size());
                    if (!of) throw SerializationError("cannot write " + path);
                }
                std::ifstream in(path, std::ios::binary);
                const ProvingKey back = deserialize_proving_key(in, z);
                const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
                const VerifyingKey &v1 = params.vk, &v2 = back.vk;
                const bool identical = !memcmp(&v1.alpha_g1, &v2.alpha_g1, 64) && !memcmp(&v1.beta_g2, &v2.beta_g2, 128) &&
                                       !memcmp(&v1.gamma_g2, &v2.gamma_g2, 128) && !memcmp(&v1.delta_g2, &v2.delta_g2, 128) &&
                                       same(v1.gamma_abc_g1, v2.gamma_abc_g1) && !memcmp(&params.beta_g1, &back.beta_g1, 64) &&
                                       !memcmp(&params.delta_g1, &back.delta_g1, 64) && same(params.a_query, back.a_query) &&
                                       same(params.b_g1_query, back.b_g1_query) && same(params.b_g2_query, back.b_g2_query) &&
                                       same(params.h_query, back.h_query) && same(params.l_query, back.l_query) &&
                                       in.tellg() == (std::streampos)bytes.size();
                std::printf("ark_keys %s bytes=%zu fnv=%016llx identical=%d, write + read %.1f ms\n", z ? "compressed" : "uncompressed",
                            bytes.size(), (unsigned long long)fnv(bytes.data(), bytes.size()), identical ? 1 : 0, ms);
            }
        }
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
}
