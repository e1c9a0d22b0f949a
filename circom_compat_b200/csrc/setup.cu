// setup.cu - b2g_setup: ark-groth16 0.5's generate_parameters_with_qap (LibsnarkReduction::instance_map_with_evaluation, and
// CircomReduction::h_query_scalars of /root/reference/src/circom/qap.rs:90-105 for the H query) on the device.
//
//   Lagrange coefficients  L_i(tau) = iNTT_n(1, tau, ..., tau^(n-1))_i   (ntt_powers + ntt_plain; tau in the domain gives
//                          ark-poly's indicator vector with no special case)
//   column sums            a_j = sum_rows A[r][j] L_r (+ L_(m+j) for the public-input rows), b_j, c_j likewise: one product per
//                          nonzero, a radix sort of the nonzeros by column and a reduce-by-key with the Fr addition, so a
//                          column shared by most rows (the constant wire) is summed by many threads
//   combination            (beta a_j + alpha b_j + c_j) / gamma for j < num_inputs, / delta for the others
//   H query                LibsnarkReduction: tau^i (tau^n - 1) / delta, i < n - 1; CircomReduction: the odd entries of the
//                          iNTT over 2n points of (delta^-1 tau^i, i < 2n - 1, then one zero)
//   group elements         fixed_base_kernel from the 8-bit window tables of the given generators, in slices through one
//                          bounded device buffer
// Every device buffer is zeroed before it is freed: all of them hold the toxic waste or values derived from it.
#include <cub/cub.cuh>
#include <algorithm>
#include <cstring>
#include <vector>
#include "../../include/b2groth.h"
#include "ec.cuh"
#include "fixed.cuh"
#include "ntt.cuh"
#include "setup.cuh"
#include "util.cuh"
#include "verify.cuh"

namespace b2g {

// constants of one setup (Fr, Montgomery unless noted), one array on the device
enum {
    K_IN = 0,                     // alpha, beta, gamma, delta, tau as given (canonical)
    K_ALPHA = 5, K_BETA, K_GINV, K_DINV, K_ONE, K_HSCALE,
    K_G1 = 11,                    // alpha, beta, delta (canonical): the scalars of alpha_g1, beta_g1, delta_g1
    K_G2 = 14,                    // beta, gamma, delta (canonical): the scalars of beta_g2, gamma_g2, delta_g2
    K_PW = 17,                    // tau^(2^b), b <= 27
    K_COUNT = K_PW + 28
};

__global__ void setup_consts_kernel(fe* __restrict__ k, int logn, int libsnark) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const fe alpha = k[K_IN], beta = k[K_IN + 1], gamma = k[K_IN + 2], delta = k[K_IN + 3];
    fe p = Fr::from_canonical(k[K_IN + 4]);
    for (int b = 0; b < 28; b++) { k[K_PW + b] = p; p = Fr::sqr(p); }
    const fe dinv = Fr::inv(Fr::from_canonical(delta));
    k[K_ALPHA] = Fr::from_canonical(alpha);
    k[K_BETA] = Fr::from_canonical(beta);
    k[K_GINV] = Fr::inv(Fr::from_canonical(gamma));
    k[K_DINV] = dinv;
    k[K_ONE] = Fr::one();
    // tau^n = k[K_PW + logn]: Z(tau) / delta for LibsnarkReduction, delta^-1 for CircomReduction
    k[K_HSCALE] = libsnark ? Fr::mul(Fr::sub(k[K_PW + logn], Fr::one()), dinv) : dinv;
    k[K_G1] = alpha; k[K_G1 + 1] = beta; k[K_G1 + 2] = delta;
    k[K_G2] = beta; k[K_G2 + 1] = gamma; k[K_G2 + 2] = delta;
}

__global__ void __launch_bounds__(256) setup_iota_kernel(uint32_t n, uint32_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = i;
}

// prod[k] = val[p] * L[row of p] for the k-th nonzero in column order, p = perm[k]; the row is found by binary search in rowptr,
// so a long row costs no thread more than log2(m) steps
__global__ void __launch_bounds__(256) setup_products_kernel(uint32_t nnz, uint32_t m, const uint32_t* __restrict__ rowptr,
                                                             const fe* __restrict__ val, const fe* __restrict__ L,
                                                             const uint32_t* __restrict__ perm, fe* __restrict__ prod) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nnz) return;
    const uint32_t p = perm[k];
    uint32_t lo = 0, hi = m - 1;                         // the last row r with rowptr[r] <= p (rowptr[m] = nnz > p)
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (rowptr[mid] <= p) lo = mid; else hi = mid - 1;
    }
    fe_store(&prod[k], Fr::mul(fe_load_nc(&val[p]), fe_load_nc(&L[lo])));
}

// sums[col[i]] = agg[i] for the *runs columns that occur
__global__ void __launch_bounds__(256) setup_scatter_kernel(uint32_t nnz, const uint32_t* __restrict__ runs, const uint32_t* __restrict__ col,
                                                            const fe* __restrict__ agg, fe* __restrict__ sums) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz || i >= *runs) return;
    fe_store(&sums[col[i]], fe_load(&agg[i]));
}

// a_j += L_(m+j) for j < num_inputs; k_j = (beta a_j + alpha b_j + c_j) / (gamma or delta); a, b, k canonical in place
__global__ void __launch_bounds__(256) setup_combine_kernel(uint32_t nv, uint32_t ni, uint32_t m, const fe* __restrict__ k,
                                                            const fe* __restrict__ L, fe* __restrict__ a, fe* __restrict__ b,
                                                            fe* __restrict__ c) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    fe aj = fe_load(&a[j]);
    if (j < ni) aj = Fr::add(aj, fe_load(&L[m + j]));
    const fe bj = fe_load(&b[j]);
    fe s = Fr::add(Fr::add(Fr::mul(k[K_BETA], aj), Fr::mul(k[K_ALPHA], bj)), fe_load(&c[j]));
    s = Fr::mul(s, k[j < ni ? K_GINV : K_DINV]);
    fe_store(&a[j], Fr::to_canonical(aj));
    fe_store(&b[j], Fr::to_canonical(bj));
    fe_store(&c[j], Fr::to_canonical(s));
}

// out[i] = in[stride * i + offset] in canonical form, i < n
__global__ void __launch_bounds__(256) setup_canonical_kernel(uint32_t n, uint32_t stride, uint32_t offset, const fe* __restrict__ in,
                                                              fe* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fe_store(&out[i], Fr::to_canonical(fe_load(&in[(size_t)stride * i + offset])));
}

struct FrAddOp {
    __device__ __forceinline__ fe operator()(const fe& a, const fe& b) const { return Fr::add(a, b); }
};

// every device buffer of one setup; each is zeroed on the stream before it is freed, on success and on error alike
struct SetupMem {
    cudaStream_t st;
    std::vector<std::pair<void*, size_t>> bufs;
    template <class T> T* alloc(size_t bytes) {
        void* p = nullptr;
        CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1));
        bufs.push_back({p, bytes ? bytes : 1});
        return (T*)p;
    }
    ~SetupMem() {
        for (auto& b : bufs) cudaMemsetAsync(b.first, 0, b.second, st);
        cudaStreamSynchronize(st);
        for (auto& b : bufs) cudaFree(b.first);
    }
};

static void secure_zero(void* p, size_t n) {
    volatile uint8_t* q = (volatile uint8_t*)p;
    while (n--) *q++ = 0;
}

// little-endian 256-bit a < m (m as 8 words)
static bool below(const uint8_t* a, const uint32_t* m) {
    for (int i = 7; i >= 0; i--) {
        uint32_t w; memcpy(&w, a + 4 * i, 4);
        if (w != m[i]) return w < m[i];
    }
    return false;
}
static const uint32_t R_WORDS[8] = {FrParams::P0, FrParams::P1, FrParams::P2, FrParams::P3, FrParams::P4, FrParams::P5, FrParams::P6, FrParams::P7};
static const uint32_t Q_WORDS[8] = {FqParams::P0, FqParams::P1, FqParams::P2, FqParams::P3, FqParams::P4, FqParams::P5, FqParams::P6, FqParams::P7};
static bool all_zero32(const uint8_t* a) { for (int i = 0; i < 32; i++) if (a[i]) return false; return true; }

constexpr size_t SETUP_SLICE = 1u << 20;                // points per fixed-base launch: bounds the output buffer to 128 MiB

// n points scalars[i] * G from the window table of G, into the caller's host buffer, in slices through d_out
template <class C, class F>
static void setup_points(const void* table, const fe* scalars, size_t n, uint8_t* d_out, void* host, cudaStream_t st) {
    const size_t aff = 2 * Bytes<F>::ELEM;
    for (size_t off = 0; off < n; off += SETUP_SLICE) {
        const size_t cnt = n - off < SETUP_SLICE ? n - off : SETUP_SLICE;
        fixed_base_kernel<C, F><<<(unsigned)((cnt + 127) / 128), 128, 0, st>>>(table, scalars + off, (uint32_t)cnt, d_out);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync((uint8_t*)host + off * aff, d_out, cnt * aff, cudaMemcpyDeviceToHost, st));
    }
}

static void setup_run(b2g_ctx* ctx, const b2g_mat_desc* d, const b2g_setup_secrets* sec, const b2g_setup_out* o) {
    if (!ctx || !d || !sec || !o) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_view(ctx);
    if (cv.proof_pending) throw_error(B2G_E_SHAPE, "a submitted proof is still pending on this context: call b2g_prove_wait first");
    const int logn = mat_desc_check(d, true);
    const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
    if (!libsnark && logn > 26) throw_error(B2G_E_DOMAIN, "PolynomialDegreeTooLarge: a CircomReduction setup transforms over 2n points, so n must fit 2^26");
    const uint32_t m = d->num_constraints, ni = d->num_inputs, nv = d->n_vars;
    const size_t n = (size_t)1 << logn, nh = libsnark ? n - 1 : n;
    if (!sec->alpha || !sec->beta || !sec->gamma || !sec->delta || !sec->tau) throw_error(B2G_E_SHAPE, "null secret");
    if (!o->alpha_g1 || !o->beta_g1 || !o->delta_g1 || !o->beta_g2 || !o->gamma_g2 || !o->delta_g2 || !o->gamma_abc_g1 || !o->a_query ||
        !o->b_g1_query || !o->b_g2_query || (nv > ni && !o->l_query) || (nh && !o->h_query))
        throw_error(B2G_E_SHAPE, "null output buffer");
    const void* secs[5] = {sec->alpha, sec->beta, sec->gamma, sec->delta, sec->tau};
    static const char* names[5] = {"alpha", "beta", "gamma", "delta", "tau"};
    for (int i = 0; i < 5; i++)
        if (!below((const uint8_t*)secs[i], R_WORDS)) throw_error(B2G_E_INPUT, std::string("secret ") + names[i] + " is not below r");
    if (all_zero32((const uint8_t*)sec->gamma)) throw_error(B2G_E_INPUT, "gamma is zero");
    if (all_zero32((const uint8_t*)sec->delta)) throw_error(B2G_E_INPUT, "delta is zero");
    for (int i = 0; i < 2; i++)
        if (sec->g1 && !below((const uint8_t*)sec->g1 + 32 * i, Q_WORDS)) throw_error(B2G_E_INPUT, "g1: coordinate not below p");
    for (int i = 0; i < 4; i++)
        if (sec->g2 && !below((const uint8_t*)sec->g2 + 32 * i, Q_WORDS)) throw_error(B2G_E_INPUT, "g2: coordinate not below p");
    const uint32_t annz = d->a_rowptr[m], bnnz = d->b_rowptr[m], cnnz = d->c_rowptr[m];
    const uint32_t maxnnz = std::max(annz, std::max(bnnz, cnnz));
    if (maxnnz > (uint32_t)INT32_MAX) throw_error(B2G_E_DEVICE, "b2g_setup: more than 2^31 - 1 nonzeros in one matrix");

    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    SetupMem mem{st, {}};
    // generators first: a bad one is refused before anything secret reaches the device
    uint8_t* d_gen = mem.alloc<uint8_t>(64 + 128);
    if (sec->g1) CUDA_CHECK(cudaMemcpyAsync(d_gen, sec->g1, 64, cudaMemcpyHostToDevice, st));
    if (sec->g2) CUDA_CHECK(cudaMemcpyAsync(d_gen + 64, sec->g2, 128, cudaMemcpyHostToDevice, st));
    switch (setup_generators_check(sec->g1 ? d_gen : nullptr, sec->g2 ? d_gen + 64 : nullptr, st)) {
        case 1: throw_error(B2G_E_INPUT, "g1 is at infinity or not on the curve");
        case 2: throw_error(B2G_E_INPUT, "g2 is at infinity or not on the twist");
        case 3: throw_error(B2G_E_INPUT, "g2 is not in G2 (the order-r subgroup of the twist)");
        default: break;
    }

    fe* d_k = mem.alloc<fe>(K_COUNT * sizeof(fe));
    {
        uint8_t h_in[5 * 32];
        for (int i = 0; i < 5; i++) memcpy(h_in + 32 * i, secs[i], 32);
        // on the setup's stream, which is not ordered with the legacy default stream; h_in is wiped once the copy is done
        cudaError_t e = cudaMemcpyAsync(d_k, h_in, sizeof(h_in), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        secure_zero(h_in, sizeof(h_in));
        CUDA_CHECK(e);
    }
    setup_consts_kernel<<<1, 1, 0, st>>>(d_k, logn, libsnark ? 1 : 0);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // Lagrange coefficients at tau; tmp also serves the 2n-point transform of the CircomReduction H query
    const size_t ntmp = libsnark ? n : 2 * n;
    fe* d_L = mem.alloc<fe>(n * sizeof(fe));
    fe* d_tmp = mem.alloc<fe>(ntmp * sizeof(fe));
    NttDomain dom;
    struct DomGuard { NttDomain& d; ~DomGuard() { ntt_domain_destroy(d); } } dg{dom};
    ntt_domain_create(dom, logn, st);
    ntt_powers(logn, d_k + K_PW, d_k + K_ONE, d_L, st);
    ntt_plain(dom, d_L, d_tmp, true, st);

    // column sums of A, B, C over the rows (Montgomery), then a, b and k = (beta a + alpha b + c) / (gamma or delta)
    fe* d_sum[3];
    for (int x = 0; x < 3; x++) {
        d_sum[x] = mem.alloc<fe>((size_t)nv * sizeof(fe));
        CUDA_CHECK(cudaMemsetAsync(d_sum[x], 0, (size_t)nv * sizeof(fe), st));
    }
    if (maxnnz) {
        int end_bit = 1;
        while (end_bit < 32 && (1ull << end_bit) < nv) end_bit++;
        uint32_t* d_rowptr = mem.alloc<uint32_t>(((size_t)m + 1) * 4);
        uint32_t* d_col = mem.alloc<uint32_t>((size_t)maxnnz * 4);
        fe* d_val = mem.alloc<fe>((size_t)maxnnz * sizeof(fe));
        uint32_t* d_keys = mem.alloc<uint32_t>((size_t)maxnnz * 4);
        uint32_t* d_idx = mem.alloc<uint32_t>((size_t)maxnnz * 4);
        uint32_t* d_perm = mem.alloc<uint32_t>((size_t)maxnnz * 4);
        fe* d_prod = mem.alloc<fe>((size_t)maxnnz * sizeof(fe));
        fe* d_agg = mem.alloc<fe>((size_t)maxnnz * sizeof(fe));
        uint32_t* d_runs = mem.alloc<uint32_t>(4);
        size_t sort_bytes = 0, reduce_bytes = 0;
        CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_col, d_keys, d_idx, d_perm, (int)maxnnz, 0, end_bit, st));
        CUDA_CHECK(cub::DeviceReduce::ReduceByKey(nullptr, reduce_bytes, d_keys, d_col, d_prod, d_agg, d_runs, FrAddOp(), (int)maxnnz, st));
        const size_t temp_bytes = std::max(sort_bytes, reduce_bytes);
        void* d_temp = mem.alloc<void>(temp_bytes);
        const uint32_t* rowptrs[3] = {d->a_rowptr, d->b_rowptr, d->c_rowptr};
        const uint32_t* cols[3] = {d->a_col, d->b_col, d->c_col};
        const void* vals[3] = {d->a_val, d->b_val, d->c_val};
        const uint32_t nnzs[3] = {annz, bnnz, cnnz};
        for (int x = 0; x < 3; x++) {
            const uint32_t nnz = nnzs[x];
            if (!nnz) continue;
            const unsigned blocks = (nnz + 255) / 256;
            CUDA_CHECK(cudaMemcpyAsync(d_rowptr, rowptrs[x], ((size_t)m + 1) * 4, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(d_col, cols[x], (size_t)nnz * 4, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(d_val, vals[x], (size_t)nnz * sizeof(fe), cudaMemcpyHostToDevice, st));
            setup_iota_kernel<<<blocks, 256, 0, st>>>(nnz, d_idx);
            size_t bytes = temp_bytes;
            CUDA_CHECK(cub::DeviceRadixSort::SortPairs(d_temp, bytes, d_col, d_keys, d_idx, d_perm, (int)nnz, 0, end_bit, st));
            setup_products_kernel<<<blocks, 256, 0, st>>>(nnz, m, d_rowptr, d_val, d_L, d_perm, d_prod);
            bytes = temp_bytes;
            // the unique columns overwrite d_col: the sort has consumed it
            CUDA_CHECK(cub::DeviceReduce::ReduceByKey(d_temp, bytes, d_keys, d_col, d_prod, d_agg, d_runs, FrAddOp(), (int)nnz, st));
            setup_scatter_kernel<<<blocks, 256, 0, st>>>(nnz, d_runs, d_col, d_agg, d_sum[x]);
            g_launch_count += 3;
            CUDA_CHECK(cudaGetLastError());
        }
    }
    setup_combine_kernel<<<(nv + 255) / 256, 256, 0, st>>>(nv, ni, m, d_k, d_L, d_sum[0], d_sum[1], d_sum[2]);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // H query scalars (canonical) in d_h
    fe* d_h = mem.alloc<fe>(n * sizeof(fe));
    if (libsnark) {
        ntt_powers(logn, d_k + K_PW, d_k + K_HSCALE, d_tmp, st);
        setup_canonical_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, 1, 0, d_tmp, d_h);
    } else {
        NttDomain dom2;
        struct Dom2Guard { NttDomain& d; ~Dom2Guard() { ntt_domain_destroy(d); } } dg2{dom2};
        ntt_domain_create(dom2, logn + 1, st);
        fe* d_hv = mem.alloc<fe>(2 * n * sizeof(fe));
        ntt_powers(logn + 1, d_k + K_PW, d_k + K_HSCALE, d_hv, st);
        CUDA_CHECK(cudaMemsetAsync(d_hv + 2 * n - 1, 0, sizeof(fe), st));          // 2n - 1 powers, padded with one zero
        ntt_plain(dom2, d_hv, d_tmp, true, st);
        setup_canonical_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, 2, 1, d_hv, d_h);
        CUDA_CHECK(cudaStreamSynchronize(st));                                     // dom2 is freed at the end of this block
    }
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // group elements
    void* d_tab1 = mem.alloc<void>(32 * 255 * 64);
    void* d_tab2 = mem.alloc<void>(32 * 255 * 128);
    fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(d_tab1, sec->g1 ? d_gen : nullptr);
    fixed_table_kernel<G2, Fq2><<<(32 * 255 + 63) / 64, 64, 0, st>>>(d_tab2, sec->g2 ? d_gen + 64 : nullptr);
    g_launch_count += 2;
    CUDA_CHECK(cudaGetLastError());
    const size_t most = std::max(std::max((size_t)nv, nh), (size_t)3);
    uint8_t* d_out = mem.alloc<uint8_t>((most < SETUP_SLICE ? most : SETUP_SLICE) * 128);
    setup_points<G1, Fq>(d_tab1, d_k + K_G1, 1, d_out, o->alpha_g1, st);
    setup_points<G1, Fq>(d_tab1, d_k + K_G1 + 1, 1, d_out, o->beta_g1, st);
    setup_points<G1, Fq>(d_tab1, d_k + K_G1 + 2, 1, d_out, o->delta_g1, st);
    setup_points<G2, Fq2>(d_tab2, d_k + K_G2, 1, d_out, o->beta_g2, st);
    setup_points<G2, Fq2>(d_tab2, d_k + K_G2 + 1, 1, d_out, o->gamma_g2, st);
    setup_points<G2, Fq2>(d_tab2, d_k + K_G2 + 2, 1, d_out, o->delta_g2, st);
    setup_points<G1, Fq>(d_tab1, d_sum[2], ni, d_out, o->gamma_abc_g1, st);
    setup_points<G1, Fq>(d_tab1, d_sum[0], nv, d_out, o->a_query, st);
    setup_points<G1, Fq>(d_tab1, d_sum[1], nv, d_out, o->b_g1_query, st);
    setup_points<G2, Fq2>(d_tab2, d_sum[1], nv, d_out, o->b_g2_query, st);
    setup_points<G1, Fq>(d_tab1, d_sum[2] + ni, nv - ni, d_out, o->l_query, st);
    setup_points<G1, Fq>(d_tab1, d_h, nh, d_out, o->h_query, st);
    CUDA_CHECK(cudaStreamSynchronize(st));
}

}  // namespace b2g

extern "C" {

int b2g_setup(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_setup_secrets* secrets, b2g_setup_out* out) {
    return b2g::guarded([&] {
        try {
            b2g::setup_run(ctx, circuit, secrets, out);
        } catch (const b2g::B2gError& e) {
            // a buffer that did not fit leaves cudaErrorMemoryAllocation as the thread's last error: clear it, so that the
            // context's next call does not fail on it
            if (e.code == B2G_E_DEVICE) cudaGetLastError();
            throw;
        }
    });
}

}  // extern "C"
