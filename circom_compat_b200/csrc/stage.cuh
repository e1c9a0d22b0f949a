// stage.cuh - what the streamed ceremony passes (ptau.cu, contribute.cu) share: the double-buffered host-to-device staging
// and the check of a 32-byte scalar.
#pragma once
#include <cstring>
#include "fp.cuh"
#include "util.cuh"

namespace b2g {

// a 32-byte little-endian scalar in [1, r)
inline bool scalar_ok(const uint8_t* a) {
    static const uint32_t R_LIMBS[8] = {FrParams::P0, FrParams::P1, FrParams::P2, FrParams::P3, FrParams::P4, FrParams::P5, FrParams::P6, FrParams::P7};
    bool zero = true;
    for (int i = 0; i < 32; i++) zero = zero && !a[i];
    if (zero) return false;
    for (int i = 7; i >= 0; i--) {
        uint32_t w; memcpy(&w, a + 4 * i, 4);
        if (w != R_LIMBS[i]) return w < R_LIMBS[i];
    }
    return false;
}

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
