// util.cuh - error plumbing shared by the host side of the library.  Exceptions never cross the C ABI: every
// extern "C" entry point catches B2gError and returns its code (include/b2groth.h).
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <atomic>
#include <cstdint>

#define B2G_OK 0
#define B2G_E_DOMAIN (-1)   /* domain larger than 2^28: SynthesisError::PolynomialDegreeTooLarge, qap.rs:31 */
#define B2G_E_SHAPE (-2)    /* inconsistent sizes / null pointers */
#define B2G_E_DEVICE (-3)   /* CUDA or NCCL failure */
#define B2G_E_INPUT (-4)    /* malformed input data (e.g. off-curve point, bad zkey) */

namespace b2g {

struct B2gError : public std::runtime_error {
    int code;
    B2gError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

extern std::atomic<uint64_t> g_launch_count;   // kernels launched by this library (defined in msm.cu)

extern thread_local std::string g_last_error;   // b2g_last_error() (defined in prover.cu)

[[noreturn]] inline void throw_error(int code, const std::string& msg) { throw B2gError(code, msg); }

#define CUDA_CHECK(expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t _e = (expr);                                                                           \
        if (_e != cudaSuccess)                                                                             \
            ::b2g::throw_error(B2G_E_DEVICE, std::string("CUDA error ") + cudaGetErrorString(_e) + " at " + \
                                                 __FILE__ + ":" + std::to_string(__LINE__) + " (" #expr ")"); \
    } while (0)

// runs the body of a C entry point: returns B2G_OK, or the error code with its message left for b2g_last_error()
template <class Fn>
inline int guarded(Fn&& fn) {
    try { fn(); return B2G_OK; }
    catch (const B2gError& e) { g_last_error = e.what(); return e.code; }
    catch (const std::exception& e) { g_last_error = e.what(); return B2G_E_DEVICE; }
    catch (...) { g_last_error = "unknown error"; return B2G_E_DEVICE; }
}

// guarded for entry points that allocate as they go: a buffer that did not fit leaves cudaErrorMemoryAllocation as the
// thread's last error; it is cleared, so that the context's next call does not fail on it
template <class Fn>
inline int guarded_clear(Fn&& fn) {
    return guarded([&] {
        try {
            fn();
        } catch (const B2gError& e) {
            if (e.code == B2G_E_DEVICE) cudaGetLastError();
            throw;
        }
    });
}

// ------------------------------------------------------------------------------------------------ host helpers
struct DevGuard {
    int prev = 0;
    explicit DevGuard(int dev) { cudaGetDevice(&prev); CUDA_CHECK(cudaSetDevice(dev)); }
    ~DevGuard() { cudaSetDevice(prev); }
};

template <class T>
inline T* dev_upload(const void* host, size_t bytes, cudaStream_t st) {
    T* d = nullptr;
    CUDA_CHECK(cudaMalloc(&d, bytes ? bytes : 1));
    if (bytes) CUDA_CHECK(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, st));
    return d;
}

}  // namespace b2g
