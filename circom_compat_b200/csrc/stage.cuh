// stage.cuh - the host helpers the setup, ceremony and key-check entry points (setup.cu, ptau.cu, contribute.cu and the
// ceremony half of verify.cu) share: the scalar and point predicates, the owners of their device, pinned and secret memory,
// their repeated preconditions, the report of a streamed pass's first bad point, and the double-buffered host-to-device staging.
#pragma once
#include <cstring>
#include <string>
#include <utility>
#include <vector>
#include "../../include/b2groth.h"
#include "fp.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {

// ------------------------------------------------------------------------------------------------ scalars and points
// the little-endian 32-bit words of r and of p
inline constexpr uint32_t R_WORDS[8] = {FrParams::P0, FrParams::P1, FrParams::P2, FrParams::P3, FrParams::P4, FrParams::P5, FrParams::P6, FrParams::P7};
inline constexpr uint32_t P_WORDS[8] = {FqParams::P0, FqParams::P1, FqParams::P2, FqParams::P3, FqParams::P4, FqParams::P5, FqParams::P6, FqParams::P7};

// a little-endian 256-bit a < m (m as 8 words)
inline bool below(const uint8_t* a, const uint32_t* m) {
    for (int i = 7; i >= 0; i--) {
        uint32_t w; memcpy(&w, a + 4 * i, 4);
        if (w != m[i]) return w < m[i];
    }
    return false;
}

inline bool all_zero(const void* p, size_t n) {
    const uint8_t* b = (const uint8_t*)p;
    for (size_t i = 0; i < n; i++) if (b[i]) return false;
    return true;
}

// a 32-byte little-endian scalar in [1, r)
inline bool scalar_ok(const uint8_t* a) { return !all_zero(a, 32) && below(a, R_WORDS); }

// ------------------------------------------------------------------------------------------------ ownership
// device buffers freed together once the stream is idle, on success and on error alike; with `zero` (buffers that hold secrets
// or values derived from them) each is zeroed on the stream first
struct DevArena {
    cudaStream_t st;
    bool zero;
    std::vector<std::pair<void*, size_t>> bufs;
    explicit DevArena(cudaStream_t s, bool zero_first = false) : st(s), zero(zero_first) {}
    DevArena(const DevArena&) = delete;
    DevArena& operator=(const DevArena&) = delete;
    template <class T = uint8_t> T* alloc(size_t bytes) {
        void* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1));
        bufs.push_back({p, bytes ? bytes : 1});
        return (T*)p;
    }
    ~DevArena() {
        if (bufs.empty()) return;
        if (zero) for (auto& b : bufs) cudaMemsetAsync(b.first, 0, b.second, st);
        cudaStreamSynchronize(st);
        for (auto& b : bufs) cudaFree(b.first);
    }
};

struct PinnedHost {
    uint8_t* p = nullptr;
    size_t bytes = 0;
    explicit PinnedHost(size_t b) : bytes(b) { CUDA_CHECK(cudaHostAlloc((void**)&p, b, cudaHostAllocDefault)); }
    PinnedHost(const PinnedHost&) = delete;
    PinnedHost& operator=(const PinnedHost&) = delete;
    ~PinnedHost() { if (p) cudaFreeHost(p); }
};

// copies the n <= 5 32-byte host secrets secs[0 .. n) to the device buffer d on the stream, which it synchronises; the host
// staging is wiped once the copy is done, on success and on error alike
inline void upload_secrets(void* d, const void* const* secs, int n, cudaStream_t st) {
    uint8_t h[5 * 32];
    for (int i = 0; i < n; i++) memcpy(h + 32 * i, secs[i], 32);
    // on the caller's stream, which is not ordered with the legacy default stream
    cudaError_t e = cudaMemcpyAsync(d, h, 32 * (size_t)n, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    volatile uint8_t* q = h;
    for (size_t i = 0; i < sizeof(h); i++) q[i] = 0;
    CUDA_CHECK(e);
}

// ------------------------------------------------------------------------------------------------ preconditions
// (the pending-proof check is ctx_idle, verify.cuh; those of a circuit are in setup.cuh)
// the ceremony's powers cover the circuit's domain of 2^logn points
inline void powers_cover(const b2g_powers_desc* pw, int logn) {
    if (pw->log_size > 28 || logn > (int)pw->log_size)
        throw_error(B2G_E_DOMAIN, "PolynomialDegreeTooLarge: the circuit's domain of 2^" + std::to_string(logn) +
                                      " points exceeds the ceremony's 2^" + std::to_string(pw->log_size) + " powers");
}

// the ceremony's arrays are given (beta_g2 only `with_beta_g2`)
inline void powers_arrays(const b2g_powers_desc* pw, bool with_beta_g2) {
    if (!pw->tau_g1 || !pw->tau_g2 || !pw->alpha_tau_g1 || !pw->beta_tau_g1 || (with_beta_g2 && !pw->beta_g2))
        throw_error(B2G_E_SHAPE, "null powers array");
}

// the buffers of a key of nv variables, ni inputs and nh H-query points are given
inline void setup_out_buffers(const b2g_setup_out* o, uint32_t nv, uint32_t ni, size_t nh) {
    if (!o->alpha_g1 || !o->beta_g1 || !o->delta_g1 || !o->beta_g2 || !o->gamma_g2 || !o->delta_g2 || !o->gamma_abc_g1 || !o->a_query ||
        !o->b_g1_query || !o->b_g2_query || (nv > ni && !o->l_query) || (nh && !o->h_query))
        throw_error(B2G_E_SHAPE, "null output buffer");
}

// tau_g1[0] and tau_g2[0] are not at infinity
inline void powers_first_finite(const b2g_powers_desc* pw) {
    if (all_zero(pw->tau_g1, 64)) throw_error(B2G_E_INPUT, "tau_g1[0]: at infinity");
    if (all_zero(pw->tau_g2, 128)) throw_error(B2G_E_INPUT, "tau_g2[0]: at infinity");
}

// ------------------------------------------------------------------------------------------------ streamed passes
// the rule that point `index` of a host array breaks (powers_point_rule; gen: index 0 must be the generator), through the device
// scratch pt (128 B) and word (4 B).  A point the pass found bad but that breaks none of the rules is B2G_E_DEVICE, named by fn.
inline uint32_t bad_point_rule(const char* fn, const void* host, uint64_t index, bool g2, bool gen, uint8_t* pt, uint32_t* word,
                               cudaStream_t st) {
    const size_t row = g2 ? 128 : 64;
    CUDA_CHECK(cudaMemcpyAsync(pt, (const uint8_t*)host + index * row, row, cudaMemcpyHostToDevice, st));
    const uint32_t rule = powers_point_rule(g2, pt, gen && index == 0, word, st);
    if (!rule || rule > 5) throw_error(B2G_E_DEVICE, std::string(fn) + ": the point rules disagree on point " + std::to_string(index));
    return rule;
}

// mont[j] = canon[j] in Montgomery form, j < n (device), in one single-thread launch (ptau.cu)
void to_mont(const fe* canon, uint32_t n, fe* mont, cudaStream_t st);

// two pinned host buffers and two device buffers of `bytes` each, a copy stream and the events that order their reuse
struct Staging {
    cudaStream_t st = nullptr, cp = nullptr;
    uint8_t *host[2] = {nullptr, nullptr}, *dev[2] = {nullptr, nullptr};
    cudaEvent_t copied[2] = {nullptr, nullptr}, used[2] = {nullptr, nullptr};
    Staging(size_t bytes, cudaStream_t s) : st(s) {
        CUDA_CHECK(cudaStreamCreateWithFlags(&cp, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            CUDA_CHECK(cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
            CUDA_CHECK(cudaEventCreateWithFlags(&used[b], cudaEventDisableTiming));
            CUDA_CHECK(cudaHostAlloc((void**)&host[b], bytes, cudaHostAllocDefault));
            CUDA_CHECK(cudaMalloc(&dev[b], bytes));
        }
    }
    // the upload of one slice of a pass: `bytes` from src through host[b] to dev[b], once the last copy out of host[b] and the
    // last use of dev[b] (the caller records used[b]) are done; st waits for it.  Returns dev[b].
    uint8_t* upload(int b, const void* src, size_t bytes) {
        CUDA_CHECK(cudaEventSynchronize(copied[b]));
        memcpy(host[b], src, bytes);
        CUDA_CHECK(cudaStreamWaitEvent(cp, used[b], 0));
        CUDA_CHECK(cudaMemcpyAsync(dev[b], host[b], bytes, cudaMemcpyHostToDevice, cp));
        CUDA_CHECK(cudaEventRecord(copied[b], cp));
        CUDA_CHECK(cudaStreamWaitEvent(st, copied[b], 0));
        return dev[b];
    }
    ~Staging() {                                       // nothing may still use a buffer when it is freed
        if (cp) cudaStreamSynchronize(cp);
        cudaStreamSynchronize(st);
        for (int b = 0; b < 2; b++) {
            if (host[b]) cudaFreeHost(host[b]);
            if (dev[b]) cudaFree(dev[b]);
            if (copied[b]) cudaEventDestroy(copied[b]);
            if (used[b]) cudaEventDestroy(used[b]);
        }
        if (cp) cudaStreamDestroy(cp);
    }
};

}  // namespace b2g
