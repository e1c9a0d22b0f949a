// verify.cu - Groth16 verification of many proofs in one device pass (b2g_vk_load / b2g_vk_free / b2g_verify_many).
//
// Device counterpart of the host verifier the reference's users call right after proving (GrothBn::process_vk +
// verify_with_processed_vk, /root/reference/src/zkey.rs:868-870, 914-916; ark-groth16 0.5.0): a proof (A, B, C) with public
// inputs x is valid iff
//     e(A, B) * e(IC[0] + sum_i x_i IC[i + 1], -gamma) * e(C, -delta) == e(alpha, beta).
// The key is prepared once on the device (b2g_vk_load): on-curve checks, e(alpha, beta), the line coefficients of the two
// fixed G2 arguments -gamma and -delta for every loop step (ark's G2Prepared), and an 8-bit window table per IC[i + 1].
// A batch then runs four kernels, one proof per thread (the parallelism comes from the batch):
//   inputs   one warp per (proof, input): x_i IC[i + 1] from the window table (32 look-ups and a warp tree)
//   prepare  parse the proof (canonical coordinates; >= p or off the curve -> invalid), sum the prepared inputs, affine
//   miller   one multi-Miller loop over (A, B), (prepared, -gamma), (C, -delta) sharing one f; only B is stepped here
//   final    the final exponentiation, compared with e(alpha, beta) -> one verdict byte
#include <cstring>
#include <string>
#include <vector>
#include "../../include/b2groth.h"
#include "fixed.cuh"
#include "pairing.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {
void msm_validate_points(const void* pts_dev, uint32_t n, bool g2, cudaStream_t st, const char* what);   // msm.cu
}
using namespace b2g;

constexpr size_t TABLE_BYTES = 32 * 255 * 64;       // one 8-bit window table of a G1 point
constexpr size_t F12_BYTES = 384;

struct b2g_vk {
    int device = 0;
    uint32_t n_public = 0;
    uint8_t* d_g1 = nullptr;       // alpha, IC[0..n_public] (G1 affine, Montgomery, 64 B each)
    uint8_t* d_g2 = nullptr;       // beta, gamma, delta (G2 affine, 128 B each)
    uint8_t* d_lines = nullptr;    // prepared lines of -gamma, then of -delta: 2 x ATE_LINES x LINE_BYTES
    uint8_t* d_eab = nullptr;      // e(alpha, beta), 384 B
    uint8_t* d_tabs = nullptr;     // window tables of IC[1..n_public], TABLE_BYTES apart
    bool gamma_inf = false, delta_inf = false;
};

namespace b2g {

// Per-proof record written by the prepare kernel: A (64 B), B (128 B), C (64 B), the prepared inputs (64 B), all affine
// Montgomery, then a word that is 1 when the proof's points parsed and lie on their curves.
constexpr size_t REC_BYTES_V = 384, REC_OK = 320;

struct VerifyBufs {
    size_t cap_count = 0, cap_inputs = 0;
    uint8_t *d_proofs = nullptr, *d_rec = nullptr, *d_f = nullptr, *d_verdict = nullptr;   // per proof
    uint8_t *d_pub = nullptr, *d_part = nullptr;                                            // per (proof, input)
};

void verify_bufs_free(VerifyBufs* v) {
    if (!v) return;
    for (void* p : {(void*)v->d_proofs, (void*)v->d_rec, (void*)v->d_f, (void*)v->d_verdict, (void*)v->d_pub, (void*)v->d_part}) if (p) cudaFree(p);
    delete v;
}

// ------------------------------------------------------------------------------------------------ kernels
// x * IC[i + 1] for one (proof, input) per warp: w = proof * n_public + i; pub = canonical scalars, part = G1 XYZZ records
__global__ void __launch_bounds__(128) verify_inputs_kernel(const uint8_t* __restrict__ tabs, const uint32_t* __restrict__ pub,
                                                            uint32_t n_public, size_t total, uint8_t* __restrict__ part) {
    __shared__ G1::Pt sh[4][32];
    const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= total) return;                                // whole warps leave together
    const uint32_t i = (uint32_t)(w % n_public);
    G1::Pt p = warp_fixed_mul<G1, Fq>(tabs + (size_t)i * TABLE_BYTES, pub + 8 * w, sh[threadIdx.x >> 5]);
    if ((threadIdx.x & 31) == 0) pt_store<Fq>(part, w, p);
}

// a canonical coordinate below p
__device__ __forceinline__ bool fe_below_p(const fe& a) {
    const uint32_t p[8] = {FqParams::P0, FqParams::P1, FqParams::P2, FqParams::P3, FqParams::P4, FqParams::P5, FqParams::P6, FqParams::P7};
    for (int i = 7; i >= 0; i--) if (a.l[i] != p[i]) return a.l[i] < p[i];
    return false;
}

__global__ void __launch_bounds__(128) verify_prepare_kernel(const uint8_t* __restrict__ proofs, const uint8_t* __restrict__ g1,
                                                             const uint8_t* __restrict__ part, uint32_t n_public, uint32_t count,
                                                             uint8_t* __restrict__ rec) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const uint8_t* pr = proofs + (size_t)j * 256;
    fe c[8];
    bool ok = true;
    for (int k = 0; k < 8; k++) { const fe v = fe_load(pr + 32 * k); ok &= fe_below_p(v); c[k] = Fq::from_canonical(v); }
    G1::Aff a, cc; G2::Aff b;
    a.x = c[0]; a.y = c[1]; b.x.c0 = c[2]; b.x.c1 = c[3]; b.y.c0 = c[4]; b.y.c1 = c[5]; cc.x = c[6]; cc.y = c[7];
    ok = ok && aff_on_curve<G1, Fq>(a) && aff_on_curve<G1, Fq>(cc) && aff_on_curve<G2, Fq2>(b);
    G1::Pt acc = G1::from_affine(aff_load<Fq>(g1, 1));   // IC[0]
    for (uint32_t i = 0; i < n_public; i++) G1::add(acc, pt_load<Fq>(part, (size_t)j * n_public + i));
    uint8_t* r = rec + (size_t)j * REC_BYTES_V;
    aff_store<Fq>(r, 0, a);
    aff_store<Fq2>(r + 64, 0, b);
    aff_store<Fq>(r + 192, 0, cc);
    aff_store<Fq>(r + 256, 0, G1::to_affine(acc));
    *reinterpret_cast<uint32_t*>(r + REC_OK) = ok;
}

__global__ void __launch_bounds__(64) verify_miller_kernel(const uint8_t* __restrict__ rec, const uint8_t* __restrict__ lines,
                                                           bool gamma_on, bool delta_on, uint32_t count, uint8_t* __restrict__ fout) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const uint8_t* r = rec + (size_t)j * REC_BYTES_V;
    if (!*reinterpret_cast<const uint32_t*>(r + REC_OK)) return;
    const G1::Aff a = aff_load<Fq>(r, 0), c = aff_load<Fq>(r + 192, 0), prep = aff_load<Fq>(r + 256, 0);
    const G2::Aff b = aff_load<Fq2>(r + 64, 0);
    G1::Aff fp[2];
    const uint8_t* fl[2];
    int nfix = 0;
    if (gamma_on && !G1::aff_is_inf(prep)) { fp[nfix] = prep; fl[nfix++] = lines; }
    if (delta_on && !G1::aff_is_inf(c)) { fp[nfix] = c; fl[nfix++] = lines + ATE_LINES * LINE_BYTES; }
    fe12 f;
    miller_loop(f, !G1::aff_is_inf(a) && !G2::aff_is_inf(b), a, b, nfix, fp, fl);
    Fq12::store(fout + (size_t)j * F12_BYTES, f);
}

__global__ void __launch_bounds__(64) verify_final_kernel(const uint8_t* __restrict__ rec, const uint8_t* __restrict__ fin,
                                                          const uint8_t* __restrict__ eab, uint32_t count, uint8_t* __restrict__ verdict) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    if (!*reinterpret_cast<const uint32_t*>(rec + (size_t)j * REC_BYTES_V + REC_OK)) { verdict[j] = 0; return; }
    fe12 e;
    Fq12::final_exponentiation(e, Fq12::load(fin + (size_t)j * F12_BYTES));
    verdict[j] = Fq12::eq(e, Fq12::load(eab));
}

// lines of -gamma (thread 0) and -delta (thread 1) for every loop step, in the order miller_loop reads them
__global__ void vk_lines_kernel(const uint8_t* __restrict__ g2, uint8_t* __restrict__ lines) {
    const int t = threadIdx.x;
    if (t > 1) return;
    const G2::Aff q = aff_load<Fq2>(g2, 1 + t);
    if (G2::aff_is_inf(q)) return;
    uint8_t* out = lines + (size_t)t * ATE_LINES * LINE_BYTES;
    g2_line_walk(q.x, Fq2::neg(q.y), [&](const fe2* c) {
        elem_store(out, c[0]); elem_store(out + 64, c[1]); elem_store(out + 128, c[2]);
        out += LINE_BYTES;
    });
}

__global__ void vk_pairing_kernel(const uint8_t* __restrict__ g1, const uint8_t* __restrict__ g2, uint8_t* __restrict__ eab) {
    fe12 e;
    pairing(e, aff_load<Fq>(g1, 0), aff_load<Fq2>(g2, 0));
    Fq12::store(eab, e);
}

// b2g_test_op ops 30-42 on Fq12 values (384 B), G1 / G2 affine points (64 / 128 B), lines (3 Fq2, 192 B) and projective
// twist points (X, Y, Z: 192 B), Montgomery
__global__ void pairing_test_kernel(int op, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe12 r;
    if (op == 37) {
        pairing(r, aff_load<Fq>(a, i), aff_load<Fq2>(b, i));
    } else if (op == 40) {
        const G1::Aff p = aff_load<Fq>(a, i);
        const G2::Aff q = aff_load<Fq2>(b, i);
        miller_loop(r, !G1::aff_is_inf(p) && !G2::aff_is_inf(q), p, q, 0, nullptr, nullptr);
    } else if (op == 41 || op == 42) {                     // one line step: out = T' (192 B) || (c0, c1, c2) (192 B)
        G2Proj t;
        const uint8_t* tp = a + (size_t)i * LINE_BYTES;
        elem_load(t.x, tp); elem_load(t.y, tp + 64); elem_load(t.z, tp + 128);
        fe2 c[3];
        if (op == 41) line_dbl(t, c);
        else { const G2::Aff q = aff_load<Fq2>(b, i); line_add(t, q.x, q.y, c); }
        uint8_t* o = out + (size_t)i * F12_BYTES;
        elem_store(o, t.x); elem_store(o + 64, t.y); elem_store(o + 128, t.z);
        for (int k = 0; k < 3; k++) elem_store(o + 192 + 64 * k, c[k]);
        return;
    } else {
        const fe12 x = Fq12::load(a + (size_t)i * F12_BYTES);
        switch (op) {
            case 30: Fq12::mul(r, x, Fq12::load(b + (size_t)i * F12_BYTES)); break;
            case 31: Fq12::sqr(r, x); break;
            case 32: Fq12::cyclotomic_sqr(r, x); break;
            case 33: case 34: case 35: Fq12::frobenius(r, x, op - 32); break;
            case 36: Fq12::final_exponentiation(r, x); break;
            case 38: Fq12::inv(r, x); break;
            default: {                                     // 39: x * (c0 + c3 w + c4 w^3)
                fe2 c[3];
                for (int k = 0; k < 3; k++) elem_load(c[k], b + (size_t)i * LINE_BYTES + 64 * k);
                r = x;
                Fq12::mul_by_034(r, c[0], c[1], c[2]);
            }
        }
    }
    Fq12::store(out + (size_t)i * F12_BYTES, r);
}

void pairing_test_op(cudaStream_t st, int op, const void* a, const void* b, size_t n, void* out) {
    if (op > 42 || !a || !out) throw_error(B2G_E_SHAPE, "bad arguments");
    const size_t sa = (op == 37 || op == 40) ? 64 : ((op == 41 || op == 42) ? LINE_BYTES : F12_BYTES);
    const size_t sb = op == 30 ? F12_BYTES : ((op == 37 || op == 40 || op == 42) ? 128 : (op == 39 ? LINE_BYTES : 0));
    if (sb && !b) throw_error(B2G_E_SHAPE, "this op needs operand b");
    if (n == 0) return;
    struct Bufs { uint8_t *a = nullptr, *b = nullptr, *o = nullptr; ~Bufs() { for (void* p : {(void*)a, (void*)b, (void*)o}) if (p) cudaFree(p); } } d;
    d.a = dev_upload<uint8_t>(a, n * sa, st);
    if (sb) d.b = dev_upload<uint8_t>(b, n * sb, st);
    CUDA_CHECK(cudaMalloc(&d.o, n * F12_BYTES));
    pairing_test_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(op, d.a, d.b, (uint32_t)n, d.o);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d.o, n * F12_BYTES, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ------------------------------------------------------------------------------------------------ host side
static void vk_release(b2g_vk* vk) {
    for (void* p : {(void*)vk->d_g1, (void*)vk->d_g2, (void*)vk->d_lines, (void*)vk->d_eab, (void*)vk->d_tabs}) if (p) cudaFree(p);
    delete vk;
}

static bool all_zero(const void* p, size_t n) {
    const uint8_t* b = (const uint8_t*)p;
    for (size_t i = 0; i < n; i++) if (b[i]) return false;
    return true;
}

// a canonical 32-byte scalar below r
static bool below_r(const uint32_t* k) {
    const uint32_t r[8] = {FrParams::P0, FrParams::P1, FrParams::P2, FrParams::P3, FrParams::P4, FrParams::P5, FrParams::P6, FrParams::P7};
    for (int i = 7; i >= 0; i--) if (k[i] != r[i]) return k[i] < r[i];
    return false;
}

// grows the context's verification buffers to `count` proofs and `inputs` (proof, input) pairs; never shrinks them.  A
// buffer set is marked empty before it is reallocated, so a failed allocation leaves the context consistent.
static void vbufs_ensure(VerifyBufs*& v, size_t count, size_t inputs) {
    if (!v) v = new VerifyBufs();
    if (count > v->cap_count) {
        for (uint8_t** p : {&v->d_proofs, &v->d_rec, &v->d_f, &v->d_verdict}) { if (*p) cudaFree(*p); *p = nullptr; }
        v->cap_count = 0;
        CUDA_CHECK(cudaMalloc(&v->d_proofs, count * 256));
        CUDA_CHECK(cudaMalloc(&v->d_rec, count * REC_BYTES_V));
        CUDA_CHECK(cudaMalloc(&v->d_f, count * F12_BYTES));
        CUDA_CHECK(cudaMalloc(&v->d_verdict, count));
        v->cap_count = count;
    }
    if (inputs > v->cap_inputs) {
        for (uint8_t** p : {&v->d_pub, &v->d_part}) { if (*p) cudaFree(*p); *p = nullptr; }
        v->cap_inputs = 0;
        CUDA_CHECK(cudaMalloc(&v->d_pub, inputs * 32));
        CUDA_CHECK(cudaMalloc(&v->d_part, inputs * 128));
        v->cap_inputs = inputs;
    }
}

}  // namespace b2g

extern "C" {

int b2g_vk_load(b2g_ctx* ctx, const b2g_vk_desc* d, b2g_vk** out) {
    return guarded([&] {
        if (!ctx || !d || !out) throw_error(B2G_E_SHAPE, "null pointer");
        if (!d->alpha_g1 || !d->beta_g2 || !d->gamma_g2 || !d->delta_g2 || !d->gamma_abc_g1) throw_error(B2G_E_SHAPE, "null verifying-key field");
        const CtxView cv = ctx_view(ctx);
        DevGuard g(cv.device);
        cudaStream_t st = cv.st;
        struct VkGuard { b2g_vk* vk = new b2g_vk(); ~VkGuard() { if (vk) { cudaDeviceSynchronize(); vk_release(vk); } } } guard;
        b2g_vk* vk = guard.vk;
        vk->device = cv.device; vk->n_public = d->n_public;
        const size_t n1 = (size_t)d->n_public + 1;
        std::vector<uint8_t> g1((1 + n1) * 64), g2(3 * 128);
        memcpy(g1.data(), d->alpha_g1, 64);
        memcpy(g1.data() + 64, d->gamma_abc_g1, n1 * 64);
        memcpy(g2.data(), d->beta_g2, 128); memcpy(g2.data() + 128, d->gamma_g2, 128); memcpy(g2.data() + 256, d->delta_g2, 128);
        vk->gamma_inf = all_zero(d->gamma_g2, 128);
        vk->delta_inf = all_zero(d->delta_g2, 128);
        vk->d_g1 = dev_upload<uint8_t>(g1.data(), g1.size(), st);
        vk->d_g2 = dev_upload<uint8_t>(g2.data(), g2.size(), st);
        // prepare_verifying_key checks every point (verifier.py); an off-curve point fails the load with B2G_E_INPUT
        msm_validate_points(vk->d_g1, (uint32_t)(1 + n1), false, st, "alpha_g1 / gamma_abc_g1");
        msm_validate_points(vk->d_g2, 3, true, st, "beta_g2 / gamma_g2 / delta_g2");
        CUDA_CHECK(cudaMalloc(&vk->d_eab, F12_BYTES));
        CUDA_CHECK(cudaMalloc(&vk->d_lines, 2 * ATE_LINES * LINE_BYTES));
        CUDA_CHECK(cudaMalloc(&vk->d_tabs, d->n_public ? d->n_public * TABLE_BYTES : 1));
        vk_pairing_kernel<<<1, 1, 0, st>>>(vk->d_g1, vk->d_g2, vk->d_eab);
        vk_lines_kernel<<<1, 32, 0, st>>>(vk->d_g2, vk->d_lines);
        for (uint32_t i = 0; i < d->n_public; i++)
            fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(vk->d_tabs + i * TABLE_BYTES, vk->d_g1 + (size_t)(2 + i) * 64);
        g_launch_count += 2 + d->n_public;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaStreamSynchronize(st));
        guard.vk = nullptr;
        *out = vk;
    });
}

int b2g_vk_free(b2g_vk* vk) {
    return guarded([&] {
        if (!vk) return;
        DevGuard g(vk->device);
        cudaDeviceSynchronize();
        vk_release(vk);
    });
}

int b2g_vk_alpha_beta(b2g_vk* vk, void* out) {
    return guarded([&] {
        if (!vk || !out) throw_error(B2G_E_SHAPE, "null pointer");
        DevGuard g(vk->device);
        CUDA_CHECK(cudaMemcpy(out, vk->d_eab, F12_BYTES, cudaMemcpyDeviceToHost));
    });
}

int b2g_verify_many(b2g_ctx* ctx, b2g_vk* vk, uint32_t count, const void* public_inputs, const void* proofs, uint8_t* verdicts_out) {
    return guarded([&] {
        if (!ctx || !vk || !proofs || !verdicts_out || (vk->n_public && !public_inputs)) throw_error(B2G_E_SHAPE, "null pointer");
        if (count == 0) throw_error(B2G_E_SHAPE, "b2g_verify_many: count must be at least 1");
        const CtxView cv = ctx_view(ctx);
        if (vk->device != cv.device) throw_error(B2G_E_SHAPE, "the verifying key belongs to another device");
        if (cv.proof_pending) throw_error(B2G_E_SHAPE, "a submitted proof is still pending on this context: call b2g_prove_wait first");
        const size_t inputs = (size_t)count * vk->n_public;
        const uint32_t* pub = (const uint32_t*)public_inputs;
        for (size_t k = 0; k < inputs; k++)
            if (!below_r(pub + 8 * k)) throw_error(B2G_E_INPUT, "public input " + std::to_string(k % vk->n_public) + " of proof " +
                                                                 std::to_string(k / vk->n_public) + " is not below the scalar field modulus r");
        DevGuard g(cv.device);
        cudaStream_t st = cv.st;
        try {
            vbufs_ensure(*cv.vbufs, count, inputs);
        } catch (const B2gError& e) {
            if (e.code != B2G_E_DEVICE) throw;
            cudaGetLastError();
            throw_error(B2G_E_DEVICE, "b2g_verify_many: the device buffers of " + std::to_string(count) +
                                      " proofs do not fit in device memory; verify fewer per call (" + e.what() + ")");
        }
        VerifyBufs& v = **cv.vbufs;
        CUDA_CHECK(cudaMemcpyAsync(v.d_proofs, proofs, (size_t)count * 256, cudaMemcpyHostToDevice, st));
        if (inputs) {
            CUDA_CHECK(cudaMemcpyAsync(v.d_pub, public_inputs, inputs * 32, cudaMemcpyHostToDevice, st));
            verify_inputs_kernel<<<(unsigned)((inputs + 3) / 4), 128, 0, st>>>(vk->d_tabs, (const uint32_t*)v.d_pub, vk->n_public, inputs, v.d_part);
        }
        verify_prepare_kernel<<<(count + 127) / 128, 128, 0, st>>>(v.d_proofs, vk->d_g1, v.d_part, vk->n_public, count, v.d_rec);
        verify_miller_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_rec, vk->d_lines, !vk->gamma_inf, !vk->delta_inf, count, v.d_f);
        verify_final_kernel<<<(count + 63) / 64, 64, 0, st>>>(v.d_rec, v.d_f, vk->d_eab, count, v.d_verdict);
        g_launch_count += 3 + (inputs ? 1 : 0);
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(verdicts_out, v.d_verdict, count, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

}  // extern "C"
