// ptau.cu - b2g_powers_check: the algebraic checks of `snarkjs powersoftau verify` over a ceremony read once from host memory,
// and b2g_powers_msm, the tableless streamed MSM it runs (msm.cuh).
//
//   streaming     each array is read in slices of POWERS_SLICE points: a host copy into one of two pinned staging buffers,
//                 an asynchronous copy to one of two device buffers on a copy stream, then the work on the context's stream.
//                 The host copy and the device copy of slice k + 1 overlap the kernels of slice k.
//   point rules   powers_rules (verify.cu) in the same pass over each slice: coordinates, curve, infinity, the generator at
//                 index 0 (points_g2_subgroup_kernel for G2), the lowest failing index per array by atomicMin
//   sums          S_X = sum_i rho^i X_i per array by powers_msm_slice, the scalars made on the device per slice
//   verdict       powers_verdict_kernel (verify.cu, with the rest of the pairing code): P_hi, P_lo and the G2 terms of
//                 include/b2groth.h, five Miller loops, one product and one final exponentiation
#include <algorithm>
#include <cstring>
#include <string>
#include "../../include/b2groth.h"
#include "msm.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {

// the one small device buffer of a check: its layout
enum : size_t {
    PV_SUMS = 0,                  // S_T, S_A, S_B (G1 XYZZ, 128 B each), S_U (G2 XYZZ, 256 B)
    PV_G1 = 640,                  // T_0, T_1, T_(2n-2), A_0, A_(n-1), B_0, B_(n-1) (affine, 64 B each)
    PV_G2 = PV_G1 + 7 * 64,       // U_0, U_1, U_(n-1), beta_2 (affine, 128 B each)
    PV_CH = PV_G2 + 4 * 128,      // rho, sigma, pi, kappa, eps (canonical)
    PV_RHO = PV_CH + 5 * 32,      // rho (Montgomery)
    PV_BAD = PV_RHO + 32,         // the lowest failing index of each of the five arrays
    PV_POINT = PV_BAD + 64,       // the point a failure names (128 B)
    PV_WORD = PV_POINT + 128,     // the verdict, or the failing point's rule
    PV_BYTES = PV_WORD + 32
};

__global__ void powers_rho_kernel(const fe* __restrict__ canon, fe* __restrict__ mont) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *mont = Fr::from_canonical(*canon);
}

template <class C, class F>
__global__ void powers_affine_kernel(const void* __restrict__ acc, void* __restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) aff_store<F>(out, 0, C::to_affine(pt_load<F>(acc, 0)));
}

static const uint32_t R_LIMBS[8] = {FrParams::P0, FrParams::P1, FrParams::P2, FrParams::P3, FrParams::P4, FrParams::P5, FrParams::P6, FrParams::P7};

// a 32-byte little-endian scalar in [1, r)
static bool scalar_ok(const uint8_t* a) {
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

struct MsmHold {
    PowersMsm m;
    cudaStream_t st;
    MsmHold(bool g2, uint64_t count, cudaStream_t s) : st(s) { powers_msm_alloc(m, g2, (uint32_t)std::min<uint64_t>(count, POWERS_SLICE)); }
    ~MsmHold() { cudaStreamSynchronize(st); powers_msm_free(m); }
};

// one pass over `count` host points: with bad, the point rules (gen: point 0 must be the generator); with msm,
// msm->acc = sum_i rho^i X_i
static void powers_pass(Staging& sg, PowersMsm* msm, bool g2, const void* host, uint64_t count, bool gen, unsigned long long* bad,
                        const fe* rho) {
    const size_t row = g2 ? 128 : 64;
    if (msm) powers_msm_reset(*msm, sg.st);
    uint64_t k = 0;
    for (uint64_t off = 0; off < count; off += POWERS_SLICE, k++) {
        const uint32_t cnt = (uint32_t)std::min<uint64_t>(POWERS_SLICE, count - off);
        const int b = (int)(k & 1);
        CUDA_CHECK(cudaEventSynchronize(sg.copied[b]));               // the pinned buffer's last copy is done
        memcpy(sg.host[b], (const uint8_t*)host + off * row, (size_t)cnt * row);
        CUDA_CHECK(cudaStreamWaitEvent(sg.cp, sg.used[b], 0));         // the device buffer's last slice is done
        CUDA_CHECK(cudaMemcpyAsync(sg.dev[b], sg.host[b], (size_t)cnt * row, cudaMemcpyHostToDevice, sg.cp));
        CUDA_CHECK(cudaEventRecord(sg.copied[b], sg.cp));
        CUDA_CHECK(cudaStreamWaitEvent(sg.st, sg.copied[b], 0));
        if (bad) powers_rules(g2, sg.dev[b], cnt, off, gen, bad, sg.st);
        if (msm) powers_msm_slice(*msm, sg.dev[b], cnt, off, rho, sg.st);
        CUDA_CHECK(cudaEventRecord(sg.used[b], sg.st));
    }
}

struct DevBuf {
    uint8_t* p = nullptr;
    explicit DevBuf(size_t bytes) { CUDA_CHECK(cudaMalloc(&p, bytes)); }
    ~DevBuf() { if (p) cudaFree(p); }
};

static void powers_msm_run(b2g_ctx* ctx, int g2, size_t n, const void* bases, const void* rho, void* out) {
    if (!ctx || !rho || !out || (n && !bases)) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_view(ctx);
    if (cv.proof_pending) throw_error(B2G_E_SHAPE, "a submitted proof is still pending on this context: call b2g_prove_wait first");
    const uint8_t* r = (const uint8_t*)rho;
    if (!scalar_ok(r) && !std::all_of(r, r + 32, [](uint8_t b) { return b == 0; })) throw_error(B2G_E_INPUT, "rho is not below r");
    const size_t row = g2 ? 128 : 64;
    if (n == 0) { memset(out, 0, row); return; }
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevBuf v(PV_BYTES);
    MsmHold h(g2 != 0, n, st);
    Staging sg(std::min<size_t>(n, POWERS_SLICE) * row, st);
    fe* d_rho = (fe*)(v.p + PV_RHO);
    CUDA_CHECK(cudaMemcpyAsync(v.p + PV_CH, rho, 32, cudaMemcpyHostToDevice, st));
    powers_rho_kernel<<<1, 1, 0, st>>>((const fe*)(v.p + PV_CH), d_rho);
    g_launch_count += 1;
    powers_pass(sg, &h.m, g2 != 0, bases, n, false, nullptr, d_rho);
    if (g2) powers_affine_kernel<G2, Fq2><<<1, 1, 0, st>>>(h.m.acc, v.p + PV_POINT);
    else powers_affine_kernel<G1, Fq><<<1, 1, 0, st>>>(h.m.acc, v.p + PV_POINT);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, v.p + PV_POINT, row, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

static void powers_check_run(b2g_ctx* ctx, const b2g_powers_desc* pw, uint32_t log_n, const void* challenges, b2g_powers_report* out) {
    if (!ctx || !pw || !challenges || !out) throw_error(B2G_E_SHAPE, "null pointer");
    memset(out, 0, sizeof(*out));
    const CtxView cv = ctx_view(ctx);
    if (cv.proof_pending) throw_error(B2G_E_SHAPE, "a submitted proof is still pending on this context: call b2g_prove_wait first");
    if (pw->log_size > 28) throw_error(B2G_E_DOMAIN, "b2g_powers_check: log_size " + std::to_string(pw->log_size) + " exceeds 28");
    if (log_n < 1 || log_n > pw->log_size)
        throw_error(B2G_E_DOMAIN, "b2g_powers_check: log_n " + std::to_string(log_n) + " is outside 1.." + std::to_string(pw->log_size));
    if (!pw->tau_g1 || !pw->tau_g2 || !pw->alpha_tau_g1 || !pw->beta_tau_g1 || !pw->beta_g2) throw_error(B2G_E_SHAPE, "null powers array");
    static const char* const CH_NAMES[5] = {"rho", "sigma", "pi", "kappa", "eps"};
    for (int k = 0; k < 5; k++)
        if (!scalar_ok((const uint8_t*)challenges + 32 * k)) throw_error(B2G_E_INPUT, std::string("challenge ") + CH_NAMES[k] + " is 0 or >= r");
    const uint64_t n = 1ull << log_n;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevBuf v(PV_BYTES);
    MsmHold h1(false, 2 * n - 1, st), h2(true, n, st);
    Staging sg(std::max<size_t>(std::min<uint64_t>(2 * n - 1, POWERS_SLICE) * 64, std::min<uint64_t>(n, POWERS_SLICE) * 128), st);
    uint8_t* V = v.p;
    const fe* d_rho = (const fe*)(V + PV_RHO);
    unsigned long long* d_bad = (unsigned long long*)(V + PV_BAD);
    const uint8_t *T = (const uint8_t*)pw->tau_g1, *U = (const uint8_t*)pw->tau_g2, *A = (const uint8_t*)pw->alpha_tau_g1,
                  *B = (const uint8_t*)pw->beta_tau_g1;
    CUDA_CHECK(cudaMemsetAsync(V + PV_BAD, 0xff, 5 * 8, st));
    CUDA_CHECK(cudaMemcpyAsync(V + PV_CH, challenges, 5 * 32, cudaMemcpyHostToDevice, st));
    const std::pair<const uint8_t*, uint64_t> g1_pts[7] = {{T, 0}, {T, 1}, {T, 2 * n - 2}, {A, 0}, {A, n - 1}, {B, 0}, {B, n - 1}};
    for (int k = 0; k < 7; k++) CUDA_CHECK(cudaMemcpyAsync(V + PV_G1 + 64 * k, g1_pts[k].first + 64 * g1_pts[k].second, 64, cudaMemcpyHostToDevice, st));
    const std::pair<const uint8_t*, uint64_t> g2_pts[4] = {{U, 0}, {U, 1}, {U, n - 1}, {(const uint8_t*)pw->beta_g2, 0}};
    for (int k = 0; k < 4; k++) CUDA_CHECK(cudaMemcpyAsync(V + PV_G2 + 128 * k, g2_pts[k].first + 128 * g2_pts[k].second, 128, cudaMemcpyHostToDevice, st));
    powers_rho_kernel<<<1, 1, 0, st>>>((const fe*)(V + PV_CH), (fe*)(V + PV_RHO));
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    struct Array { const uint8_t* host; uint64_t count; bool g2, gen; PowersMsm* msm; size_t sum; };
    const Array arrays[5] = {{T, 2 * n - 1, false, true, &h1.m, 0}, {U, n, true, true, &h2.m, 384}, {A, n, false, false, &h1.m, 128},
                             {B, n, false, false, &h1.m, 256}, {(const uint8_t*)pw->beta_g2, 1, true, false, nullptr, 0}};
    for (int a = 0; a < 5; a++) {
        const Array& x = arrays[a];
        powers_pass(sg, x.msm, x.g2, x.host, x.count, x.gen, d_bad + a, d_rho);
        if (x.msm) CUDA_CHECK(cudaMemcpyAsync(V + PV_SUMS + x.sum, x.msm->acc, x.g2 ? 256 : 128, cudaMemcpyDeviceToDevice, st));
        uint64_t bad = 0;
        CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad + a, 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        if (bad >= x.count) continue;
        // the first failing point of the first array with one: the first rule it breaks
        const size_t row = x.g2 ? 128 : 64;
        CUDA_CHECK(cudaMemcpyAsync(V + PV_POINT, x.host + bad * row, row, cudaMemcpyHostToDevice, st));
        const uint32_t rule = powers_point_rule(x.g2, V + PV_POINT, x.gen && bad == 0, (uint32_t*)(V + PV_WORD), st);
        if (!rule) throw_error(B2G_E_DEVICE, "b2g_powers_check: the point rules disagree on point " + std::to_string(bad));
        out->ok = 0; out->rule = (uint8_t)rule; out->array = (uint8_t)a; out->index = bad;
        return;
    }
    powers_verdict(V + PV_SUMS, V + PV_G1, V + PV_G2, V + PV_CH, log_n, (uint32_t*)(V + PV_WORD), st);
    uint32_t verdict = 0;
    CUDA_CHECK(cudaMemcpyAsync(&verdict, V + PV_WORD, 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    out->ok = verdict ? 1 : 0;
    out->rule = verdict ? 0 : 6;
}

}  // namespace b2g

extern "C" {

int b2g_powers_msm(b2g_ctx* ctx, int g2, size_t n, const void* bases, const void* rho_canon, void* out_affine) {
    return b2g::guarded_clear([&] { b2g::powers_msm_run(ctx, g2, n, bases, rho_canon, out_affine); });
}

int b2g_powers_check(b2g_ctx* ctx, const b2g_powers_desc* powers, uint32_t log_n, const void* challenges, b2g_powers_report* out) {
    return b2g::guarded_clear([&] { b2g::powers_check_run(ctx, powers, log_n, challenges, out); });
}

}  // extern "C"
