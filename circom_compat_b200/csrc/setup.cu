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
//
// b2g_setup_from_powers makes the same key (gamma = delta = 1) from the points of a powers-of-tau ceremony instead, with no
// scalar known to anyone:
//   Lagrange points        [L_r] = iNTT_n(tau^i G)_r over points (points_intt: one launch per radix-2 DIF stage, one butterfly
//                          per thread, the twiddle product a variable-base double-and-add on an XYZZ record; then a gather
//                          from bit-reversed order that scales by n^-1 and converts to affine), for tau G1, tau G2, alpha tau G1
//                          and beta tau G1
//   column sums            the nonzeros sorted by column as above, then products coefficient x Lagrange point summed in pieces
//                          of PIECE_PRODUCTS per thread and reduced by column, PIECE_SUMS points per thread and level, until each
//                          column has one point; a coefficient above r / 2 multiplies the negated point by r - k
//   H query                LibsnarkReduction: tau^(i + n) G - tau^i G; CircomReduction: 1/2 iNTT_n of
//                          y_i = omega_2n^-i (tau^i G - tau^(i + n) G), the odd entries of the 2n-point transform folded
//                          into one n-point transform
// b2g_delta_update multiplies delta by x and the L and H queries by x^-1, one point per thread.
#include <cub/cub.cuh>
#include <algorithm>
#include <cstring>
#include <vector>
#include "../../include/b2groth.h"
#include "ec.cuh"
#include "fixed.cuh"
#include "ntt.cuh"
#include "setup.cuh"
#include "stage.cuh"
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

// prod[k] = val[p] * L[row of p] for the k-th nonzero in column order, p = perm[k]
__global__ void __launch_bounds__(256) setup_products_kernel(uint32_t nnz, uint32_t m, const uint32_t* __restrict__ rowptr,
                                                             const fe* __restrict__ val, const fe* __restrict__ L,
                                                             const uint32_t* __restrict__ perm, fe* __restrict__ prod) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nnz) return;
    const uint32_t p = perm[k], row = mat_row(rowptr, m, p);
    fe_store(&prod[k], Fr::mul(fe_load_nc(&val[p]), fe_load_nc(&L[row])));
}

// out[keys[i]] = agg[i] for the *runs keys that occur
__global__ void __launch_bounds__(256) scatter_sums_kernel(uint32_t n, const uint32_t* __restrict__ runs, const uint32_t* __restrict__ keys,
                                                           const fe* __restrict__ agg, fe* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || i >= *runs) return;
    fe_store(&out[keys[i]], fe_load(&agg[i]));
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

void sum_by_key(void* temp, size_t& temp_bytes, const uint32_t* keys, uint32_t* uniq, const fe* prod, fe* agg, uint32_t* runs,
                uint32_t n, fe* out, cudaStream_t st) {
    CUDA_CHECK(cub::DeviceReduce::ReduceByKey(temp, temp_bytes, keys, uniq, prod, agg, runs, FrAddOp(), (int)n, st));
    if (!temp) return;
    scatter_sums_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, runs, uniq, agg, out);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

// the nonzeros of one matrix in column order: keys = the sorted columns (from col, which the sort consumes, under nv columns) and
// perm = the nonzeros' indices in that order, through idx.  With temp null, only sets temp_bytes.
static void sort_by_column(void* temp, size_t& temp_bytes, uint32_t* col, uint32_t* keys, uint32_t* idx, uint32_t* perm, uint32_t nnz,
                           uint32_t nv, cudaStream_t st) {
    int end_bit = 1;
    while (end_bit < 32 && (1ull << end_bit) < nv) end_bit++;
    if (temp) {
        setup_iota_kernel<<<(nnz + 255) / 256, 256, 0, st>>>(nnz, idx);
        g_launch_count += 1;
    }
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, col, keys, idx, perm, (int)nnz, 0, end_bit, st));
}

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
    const CtxView cv = ctx_idle(ctx);
    const int logn = setup_domain(d);
    const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
    const uint32_t m = d->num_constraints, ni = d->num_inputs, nv = d->n_vars;
    const size_t n = (size_t)1 << logn, nh = libsnark ? n - 1 : n;
    if (!sec->alpha || !sec->beta || !sec->gamma || !sec->delta || !sec->tau) throw_error(B2G_E_SHAPE, "null secret");
    setup_out_buffers(o, nv, ni, nh);
    const void* secs[5] = {sec->alpha, sec->beta, sec->gamma, sec->delta, sec->tau};
    static const char* names[5] = {"alpha", "beta", "gamma", "delta", "tau"};
    for (int i = 0; i < 5; i++)
        if (!below((const uint8_t*)secs[i], R_WORDS)) throw_error(B2G_E_INPUT, std::string("secret ") + names[i] + " is not below r");
    if (all_zero(sec->gamma, 32)) throw_error(B2G_E_INPUT, "gamma is zero");
    if (all_zero(sec->delta, 32)) throw_error(B2G_E_INPUT, "delta is zero");
    for (int i = 0; i < 2; i++)
        if (sec->g1 && !below((const uint8_t*)sec->g1 + 32 * i, P_WORDS)) throw_error(B2G_E_INPUT, "g1: coordinate not below p");
    for (int i = 0; i < 4; i++)
        if (sec->g2 && !below((const uint8_t*)sec->g2 + 32 * i, P_WORDS)) throw_error(B2G_E_INPUT, "g2: coordinate not below p");
    const uint32_t maxnnz = max_nnz(d, "b2g_setup");

    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st, true);
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
    upload_secrets(d_k, secs, 5, st);
    setup_consts_kernel<<<1, 1, 0, st>>>(d_k, logn, libsnark ? 1 : 0);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // Lagrange coefficients at tau; tmp also serves the 2n-point transform of the CircomReduction H query
    const size_t ntmp = libsnark ? n : 2 * n;
    fe* d_L = mem.alloc<fe>(n * sizeof(fe));
    fe* d_tmp = mem.alloc<fe>(ntmp * sizeof(fe));
    NttDomainHold dom(logn, st);
    ntt_powers(logn, d_k + K_PW, d_k + K_ONE, d_L, st);
    ntt_plain(dom, d_L, d_tmp, true, st);

    // column sums of A, B, C over the rows (Montgomery), then a, b and k = (beta a + alpha b + c) / (gamma or delta)
    fe* d_sum[3];
    for (int x = 0; x < 3; x++) {
        d_sum[x] = mem.alloc<fe>((size_t)nv * sizeof(fe));
        CUDA_CHECK(cudaMemsetAsync(d_sum[x], 0, (size_t)nv * sizeof(fe), st));
    }
    if (maxnnz) {
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
        sort_by_column(nullptr, sort_bytes, d_col, d_keys, d_idx, d_perm, maxnnz, nv, st);
        sum_by_key(nullptr, reduce_bytes, d_keys, d_col, d_prod, d_agg, d_runs, maxnnz, nullptr, st);
        const size_t temp_bytes = std::max(sort_bytes, reduce_bytes);
        void* d_temp = mem.alloc<void>(temp_bytes);
        for (int x = 0; x < 3; x++) {
            const uint32_t nnz = mat_nnz(d, x);
            if (!nnz) continue;
            mat_upload(d, x, d_rowptr, d_col, d_val, st);
            size_t bytes = temp_bytes;
            sort_by_column(d_temp, bytes, d_col, d_keys, d_idx, d_perm, nnz, nv, st);
            setup_products_kernel<<<(nnz + 255) / 256, 256, 0, st>>>(nnz, m, d_rowptr, d_val, d_L, d_perm, d_prod);
            g_launch_count += 1;
            bytes = temp_bytes;
            // the unique columns overwrite d_col: the sort has consumed it
            sum_by_key(d_temp, bytes, d_keys, d_col, d_prod, d_agg, d_runs, nnz, d_sum[x], st);
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
        NttDomainHold dom2(logn + 1, st);
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

// ---------------------------------------------------------------------------------------------- points of a ceremony
constexpr uint32_t PIECE_PRODUCTS = 4;                  // products one thread sums at the first level of a column sum
constexpr uint32_t PIECE_SUMS = 32;                     // points one thread sums at each later level

// k P for an affine P and a canonical 256-bit k: mixed double-and-add from the top set bit; every exceptional case is madd's
template <class C>
__device__ __noinline__ typename C::Pt aff_mul(const typename C::Aff& p, const uint32_t* k) {
    typename C::Pt acc = C::infinity();
    if (C::aff_is_inf(p)) return acc;
    int top = 255;
    while (top >= 0 && !((k[top >> 5] >> (top & 31)) & 1u)) top--;
    #pragma unroll 1
    for (int i = top; i >= 0; i--) {
        acc = C::dbl(acc);
        if ((k[i >> 5] >> (i & 31)) & 1u) C::madd(acc, p);
    }
    return acc;
}

template <class C, class F>
__global__ void __launch_bounds__(128) pts_from_affine_kernel(const void* __restrict__ aff, uint32_t n, void* __restrict__ pts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pt_store<F>(pts, i, C::from_affine(aff_load<F>(aff, i)));
}

// one radix-2 DIF stage of the inverse transform over n = 2^logn points, half-size h = 2^s, one butterfly per thread:
//   (u, v) -> (u + v, (u - v) omega_n^-e),  e = j 2^(logn - 1 - s) for the butterfly's offset j < h in its block
// with omega_n^-e = -tw[n - 2e] for e > 0 (tw[k] = omega_2n^k, NttDomain), so the product is (v - u) tw[n - 2e]
template <class C, class F>
__global__ void __launch_bounds__(128) pts_intt_stage_kernel(void* __restrict__ pts, int logn, int s, const fe* __restrict__ tw) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (1u << (logn - 1))) return;
    const uint32_t h = 1u << s, j = t & (h - 1), i0 = ((t >> s) << (s + 1)) | j, i1 = i0 + h;
    const uint32_t e = j << (logn - 1 - s);
    const typename C::Pt u = pt_load<F>(pts, i0);
    typename C::Pt v = pt_load<F>(pts, i1), sum = u;
    C::add(sum, v);
    C::add(v, C::neg(u));                                                  // v - u
    if (e) {
        const fe k = Fr::to_canonical(fe_load_nc(&tw[(1u << logn) - 2 * e]));
        v = C::mul_scalar(v, k.l);
    } else {
        v = C::neg(v);
    }
    pt_store<F>(pts, i0, sum);
    pt_store<F>(pts, i1, v);
}

// out[k] = scale x pts[bitrev(k)] in affine form: the natural order of the DIF output, times n^-1 (or (2n)^-1)
template <class C, class F>
__global__ void __launch_bounds__(128) pts_intt_finish_kernel(const void* __restrict__ pts, int logn, const fe* __restrict__ scale,
                                                              void* __restrict__ out) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (1u << logn)) return;
    const uint32_t src = logn ? __brev(k) >> (32 - logn) : 0u;
    const fe sc = *scale;
    aff_store<F>(out, k, C::to_affine(C::mul_scalar(pt_load<F>(pts, src), sc.l)));
}

// sc[0] = n^-1, sc[1] = (2n)^-1 (canonical) from ninv = n^-1 (Montgomery)
__global__ void pts_scale_kernel(const fe* __restrict__ ninv, fe* __restrict__ sc) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe two = fe_zero(); two.l[0] = 2;
    sc[0] = Fr::to_canonical(*ninv);
    sc[1] = Fr::to_canonical(Fr::mul(*ninv, Fr::inv(Fr::from_canonical(two))));
}

// the natural-order inverse transform of the XYZZ records at pts (n = 2^logn >= 2, in place through the DIF stages), times
// *scale, to the affine points at out
template <class C, class F>
static void points_intt(const NttDomain& dom, void* pts, const fe* scale, void* out, cudaStream_t st) {
    const int logn = dom.logn;
    const uint32_t n = 1u << logn;
    for (int s = logn - 1; s >= 0; s--)
        pts_intt_stage_kernel<C, F><<<(n / 2 + 127) / 128, 128, 0, st>>>(pts, logn, s, dom.tw);
    pts_intt_finish_kernel<C, F><<<(n + 127) / 128, 128, 0, st>>>(pts, logn, scale, out);
    g_launch_count += logn + 1;
    CUDA_CHECK(cudaGetLastError());
}

// LibsnarkReduction's H query: out[i] = tau[i + n] - tau[i], i < n - 1
__global__ void __launch_bounds__(128) hq_libsnark_kernel(const void* __restrict__ tau, uint32_t n, void* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 >= n) return;
    G1::Aff a = aff_load<Fq>(tau, i);
    if (!G1::aff_is_inf(a)) a.y = Fq::neg(a.y);
    G1::Pt p = G1::from_affine(aff_load<Fq>(tau, i + n));
    G1::madd(p, a);
    aff_store<Fq>(out, i, G1::to_affine(p));
}

// CircomReduction's folded input: pts[i] = omega_2n^-i (tau[i] - tau[i + n]) = tw[n - i] (tau[i + n] - tau[i]) for i > 0,
// tau[0] - tau[n] for i = 0, with tau[2n - 1] taken as infinity
__global__ void __launch_bounds__(128) hq_circom_kernel(const void* __restrict__ tau, uint32_t n, const fe* __restrict__ tw,
                                                        void* __restrict__ pts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1::Aff a = aff_load<Fq>(tau, i);
    if (!G1::aff_is_inf(a)) a.y = Fq::neg(a.y);
    G1::Pt p = i + n < 2 * n - 1 ? G1::from_affine(aff_load<Fq>(tau, i + n)) : G1::infinity();
    G1::madd(p, a);
    if (i) {
        const fe k = Fr::to_canonical(fe_load_nc(&tw[n - i]));
        p = G1::mul_scalar(p, k.l);
    } else {
        p = G1::neg(p);
    }
    pt_store<Fq>(pts, i, p);
}

// colptr[j] = the first k with keys[k] >= j, j <= nv (keys sorted)
__global__ void __launch_bounds__(256) colptr_kernel(uint32_t nnz, uint32_t nv, const uint32_t* __restrict__ keys, uint32_t* __restrict__ colptr) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > nv) return;
    uint32_t lo = 0, hi = nnz;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (keys[mid] < j) lo = mid + 1; else hi = mid;
    }
    colptr[j] = lo;
}

// the column j < nv whose pieces ptr[j] .. ptr[j + 1] - 1 hold piece q (ptr nondecreasing, ptr[nv] > q)
__device__ __forceinline__ uint32_t piece_column(const uint32_t* __restrict__ ptr, uint32_t nv, uint32_t q) {
    uint32_t lo = 0, hi = nv - 1;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (ptr[mid] <= q) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// first level of a column sum: piece q of column j sums up to PIECE_PRODUCTS products val[p] base[row of p] of the
// column's nonzeros in sorted order (p = perm[k]); a coefficient k > r - k multiplies the negated point by r - k
template <class C, class F>
__global__ void __launch_bounds__(128) colsum_products_kernel(uint32_t pieces, uint32_t nv, uint32_t m, const uint32_t* __restrict__ rowptr,
                                                              const fe* __restrict__ val, const uint32_t* __restrict__ perm,
                                                              const uint32_t* __restrict__ colptr, const uint32_t* __restrict__ ptr,
                                                              const void* __restrict__ base, void* __restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= pieces) return;
    const uint32_t j = piece_column(ptr, nv, q);
    const uint32_t start = colptr[j] + (q - ptr[j]) * PIECE_PRODUCTS, end = min(start + PIECE_PRODUCTS, colptr[j + 1]);
    typename C::Pt acc = C::infinity();
    for (uint32_t k = start; k < end; k++) {
        const uint32_t p = perm[k], row = mat_row(rowptr, m, p);
        fe c = Fr::to_canonical(fe_load_nc(&val[p]));
        typename C::Aff b = aff_load<F>(base, row);
        const fe nc = Fr::neg(c);
        bool big = false;
        for (int w = 7; w >= 0; w--) if (c.l[w] != nc.l[w]) { big = c.l[w] > nc.l[w]; break; }
        if (big && !C::aff_is_inf(b)) { c = nc; b.y = F::neg(b.y); }
        C::add(acc, aff_mul<C>(b, c.l));
    }
    pt_store<F>(out, q, acc);
}

// a later level: piece q of column j sums up to PIECE_SUMS of the column's records of the level below (ptr_in)
template <class C, class F>
__global__ void __launch_bounds__(128) colsum_reduce_kernel(uint32_t pieces, uint32_t nv, const uint32_t* __restrict__ ptr_in,
                                                            const uint32_t* __restrict__ ptr, const void* __restrict__ in, void* __restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= pieces) return;
    const uint32_t j = piece_column(ptr, nv, q);
    const uint32_t start = ptr_in[j] + (q - ptr[j]) * PIECE_SUMS, end = min(start + PIECE_SUMS, ptr_in[j + 1]);
    typename C::Pt acc = pt_load<F>(in, start);
    for (uint32_t k = start + 1; k < end; k++) C::add(acc, pt_load<F>(in, k));
    pt_store<F>(out, q, acc);
}

// acc[j] += in[ptr[j]] for the columns with a piece at the last level (at most one each)
template <class C, class F>
__global__ void __launch_bounds__(128) colsum_accumulate_kernel(uint32_t nv, const uint32_t* __restrict__ ptr, const void* __restrict__ in,
                                                                void* __restrict__ acc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv || ptr[j + 1] == ptr[j]) return;
    typename C::Pt a = pt_load<F>(acc, j);
    C::add(a, pt_load<F>(in, ptr[j]));
    pt_store<F>(acc, j, a);
}

// out[j] = acc[j] (+ extra[m + j] for j < ni when extra is given), affine
template <class C, class F>
__global__ void __launch_bounds__(128) colsum_finish_kernel(uint32_t nv, uint32_t ni, uint32_t m, const void* __restrict__ acc,
                                                            const void* __restrict__ extra, void* __restrict__ out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    typename C::Pt a = pt_load<F>(acc, j);
    if (extra && j < ni) C::madd(a, aff_load<F>(extra, (size_t)m + j));
    aff_store<F>(out, j, C::to_affine(a));
}

// one matrix on the device with its nonzeros in column order (perm) and the pieces of every level of its column sums: level
// l >= 1 gives column j the pieces ptr[l][j] .. ptr[l][j + 1] - 1; ptr[0] is the column pointer of the sorted nonzeros.  The
// last level has at most one piece per column.
struct ColPlan {
    uint32_t nnz = 0;
    const uint32_t* rowptr = nullptr;
    const fe* val = nullptr;
    const uint32_t* perm = nullptr;
    std::vector<const uint32_t*> ptr;
    std::vector<uint32_t> pieces;
};

static ColPlan col_plan(DevArena& mem, const b2g_mat_desc* d, int x, uint32_t nv, cudaStream_t st) {
    const uint32_t m = d->num_constraints;
    ColPlan cp;
    cp.nnz = mat_nnz(d, x);
    if (!cp.nnz) return cp;
    const uint32_t nnz = cp.nnz;
    uint32_t* d_rowptr = mem.alloc<uint32_t>(((size_t)m + 1) * 4);
    uint32_t* d_col = mem.alloc<uint32_t>((size_t)nnz * 4);
    fe* d_val = mem.alloc<fe>((size_t)nnz * sizeof(fe));
    uint32_t* d_keys = mem.alloc<uint32_t>((size_t)nnz * 4);
    uint32_t* d_idx = mem.alloc<uint32_t>((size_t)nnz * 4);
    uint32_t* d_perm = mem.alloc<uint32_t>((size_t)nnz * 4);
    uint32_t* d_colptr = mem.alloc<uint32_t>(((size_t)nv + 1) * 4);
    size_t sort_bytes = 0;
    sort_by_column(nullptr, sort_bytes, d_col, d_keys, d_idx, d_perm, nnz, nv, st);
    void* d_temp = mem.alloc<void>(sort_bytes);
    mat_upload(d, x, d_rowptr, d_col, d_val, st);
    sort_by_column(d_temp, sort_bytes, d_col, d_keys, d_idx, d_perm, nnz, nv, st);
    colptr_kernel<<<(nv + 256) / 256, 256, 0, st>>>(nnz, nv, d_keys, d_colptr);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    std::vector<uint32_t> cur(nv + 1);
    CUDA_CHECK(cudaMemcpyAsync(cur.data(), d_colptr, ((size_t)nv + 1) * 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    cp.rowptr = d_rowptr; cp.val = d_val; cp.perm = d_perm;
    cp.ptr.push_back(d_colptr);
    cp.pieces.push_back(nnz);
    // the pieces of each level on the host, from the counts of the level below, until no column has more than one
    for (uint32_t per = PIECE_PRODUCTS, most = 2; most > 1; per = PIECE_SUMS) {
        std::vector<uint32_t> next(nv + 1, 0);
        most = 0;
        for (uint32_t j = 0; j < nv; j++) {
            const uint32_t c = (cur[j + 1] - cur[j] + per - 1) / per;
            next[j + 1] = next[j] + c;
            most = std::max(most, c);
        }
        uint32_t* d_ptr = mem.alloc<uint32_t>(((size_t)nv + 1) * 4);
        CUDA_CHECK(cudaMemcpyAsync(d_ptr, next.data(), ((size_t)nv + 1) * 4, cudaMemcpyHostToDevice, st));
        CUDA_CHECK(cudaStreamSynchronize(st));                         // `next` is freed at the end of this iteration
        cp.ptr.push_back(d_ptr);
        cp.pieces.push_back(next[nv]);
        cur.swap(next);
    }
    return cp;
}

// acc[j] += sum over the nonzeros (r, j, k) of the plan's matrix of k base[r] (XYZZ accumulators, one per column), through
// the scratch areas x and y (each at least cp.pieces[1] records)
template <class C, class F>
static void col_sums(const ColPlan& cp, uint32_t nv, uint32_t m, const void* base, uint8_t* x, uint8_t* y, void* acc, cudaStream_t st) {
    if (!cp.nnz) return;
    colsum_products_kernel<C, F><<<(cp.pieces[1] + 127) / 128, 128, 0, st>>>(cp.pieces[1], nv, m, cp.rowptr, cp.val, cp.perm, cp.ptr[0],
                                                                              cp.ptr[1], base, x);
    for (size_t l = 2; l < cp.ptr.size(); l++) {
        colsum_reduce_kernel<C, F><<<(cp.pieces[l] + 127) / 128, 128, 0, st>>>(cp.pieces[l], nv, cp.ptr[l - 1], cp.ptr[l], x, y);
        std::swap(x, y);
    }
    colsum_accumulate_kernel<C, F><<<(nv + 127) / 128, 128, 0, st>>>(nv, cp.ptr.back(), x, acc);
    g_launch_count += cp.ptr.size();
    CUDA_CHECK(cudaGetLastError());
}

// copies n affine points (row bytes each) to the device buffer d and refuses the array when one of them is off its curve, has a
// coordinate >= p or (subgroup) lies outside G2; `name` names the array in the message and `base` is the index of host[0] in it
static void check_upload(const char* name, uint64_t base, const void* host, size_t n, bool g2, bool subgroup, uint8_t* d, cudaStream_t st) {
    const size_t row = g2 ? 128 : 64;
    CUDA_CHECK(cudaMemcpyAsync(d, host, n * row, cudaMemcpyHostToDevice, st));
    int why = 0;
    const uint64_t bad = points_check(g2, d, n, subgroup, st, &why);
    if (bad < n)
        throw_error(B2G_E_INPUT, std::string(name) + "[" + std::to_string(base + bad) + "]: " +
                                     (why == 2 ? "not in G2" : g2 ? "off the twist or a coordinate >= p" : "off the curve or a coordinate >= p"));
}

// uploads n affine points into a new buffer of `mem`, refused as check_upload refuses them
static uint8_t* powers_upload(DevArena& mem, const char* name, const void* host, size_t n, bool g2, bool subgroup, cudaStream_t st,
                              uint64_t base = 0) {
    uint8_t* d = mem.alloc<uint8_t>(n * (g2 ? 128 : 64));
    check_upload(name, base, host, n, g2, subgroup, d, st);
    return d;
}

// CircomReduction's H query from a Lagrange block: k[i] = -(2n)^-1 omega_2n^(2i+1) (canonical), i < n, from tw[j] = omega_2n^j
// (j < n, Montgomery; omega_2n^(j+n) = -omega_2n^j) and inv2n = (2n)^-1 (canonical)
__global__ void __launch_bounds__(256) hq_lagrange_scalars_kernel(uint32_t n, const fe* __restrict__ tw, const fe* __restrict__ inv2n,
                                                                  fe* __restrict__ k) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t e = 2 * i + 1;
    const fe w = e < n ? fe_load_nc(&tw[e]) : Fr::neg(fe_load_nc(&tw[e - n]));
    fe_store(&k[i], Fr::neg(Fr::mul(w, *inv2n)));
}

// out[i] = blk[2i + 1] (+ corr[i] when corr is given), i < n
__global__ void __launch_bounds__(128) hq_lagrange_kernel(const void* __restrict__ blk, uint32_t n, const void* __restrict__ corr,
                                                          void* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1::Pt p = G1::from_affine(aff_load<Fq>(blk, 2 * (size_t)i + 1));
    if (corr) G1::madd(p, aff_load<Fq>(corr, i));
    aff_store<Fq>(out, i, G1::to_affine(p));
}

// b2g_setup_from_powers, or with lg b2g_setup_from_lagrange: the Lagrange points and the CircomReduction H query read from
// the prepared sections instead of transformed
static void setup_from_powers_run(b2g_ctx* ctx, const b2g_mat_desc* d, const b2g_powers_desc* pw, const b2g_setup_out* o,
                                  const b2g_lagrange_desc* lg = nullptr) {
    if (!ctx || !d || !pw || !o) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    const int logn = setup_domain(d);
    const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
    powers_cover(pw, logn);
    powers_arrays(pw, true);
    if (lg) {
        if (!lg->tau_g1 || !lg->tau_g2 || !lg->alpha_tau_g1 || !lg->beta_tau_g1) throw_error(B2G_E_SHAPE, "null Lagrange array");
        if (lg->log_size > 26 || lg->log_size > pw->log_size)
            throw_error(B2G_E_DOMAIN, "b2g_setup_from_lagrange: Lagrange sections of power " + std::to_string(lg->log_size) +
                                          " exceed 26 or the ceremony's power " + std::to_string(pw->log_size));
        if (logn > (int)lg->log_size)
            throw_error(B2G_E_DOMAIN, "PolynomialDegreeTooLarge: the circuit's domain of 2^" + std::to_string(logn) +
                                          " points exceeds the Lagrange sections' 2^" + std::to_string(lg->log_size));
    }
    const uint32_t m = d->num_constraints, ni = d->num_inputs, nv = d->n_vars;
    const size_t n = (size_t)1 << logn, nh = libsnark ? n - 1 : n;
    setup_out_buffers(o, nv, ni, nh);
    max_nnz(d, "b2g_setup_from_powers");

    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st, true);
    uint8_t* d_tau1 = powers_upload(mem, "tau_g1", pw->tau_g1, 2 * n - 1, false, false, st);
    uint8_t* d_tau2 = powers_upload(mem, "tau_g2", pw->tau_g2, n, true, true, st);
    uint8_t* d_atau = powers_upload(mem, "alpha_tau_g1", pw->alpha_tau_g1, n, false, false, st);
    uint8_t* d_btau = powers_upload(mem, "beta_tau_g1", pw->beta_tau_g1, n, false, false, st);
    powers_upload(mem, "beta_g2", pw->beta_g2, 1, true, true, st);
    powers_first_finite(pw);

    // the Lagrange points: four transforms through one XYZZ work area
    NttDomainHold dom(logn, st);
    fe* d_sc = mem.alloc<fe>(2 * sizeof(fe));
    pts_scale_kernel<<<1, 1, 0, st>>>(dom.ct, d_sc);                       // ct[0] = n^-1
    g_launch_count += 1;
    const unsigned pblocks = (unsigned)((n + 127) / 128);
    uint8_t *d_work = nullptr, *d_L1, *d_L2, *d_aL, *d_bL;
    if (lg) {
        // block log_n of each section, at its offset n - 1
        d_L1 = powers_upload(mem, "lagrange_tau_g1", (const uint8_t*)lg->tau_g1 + (n - 1) * 64, n, false, false, st, n - 1);
        d_L2 = powers_upload(mem, "lagrange_tau_g2", (const uint8_t*)lg->tau_g2 + (n - 1) * 128, n, true, true, st, n - 1);
        d_aL = powers_upload(mem, "lagrange_alpha_tau_g1", (const uint8_t*)lg->alpha_tau_g1 + (n - 1) * 64, n, false, false, st, n - 1);
        d_bL = powers_upload(mem, "lagrange_beta_tau_g1", (const uint8_t*)lg->beta_tau_g1 + (n - 1) * 64, n, false, false, st, n - 1);
    } else {
        d_work = mem.alloc<uint8_t>(n * 256);
        d_L1 = mem.alloc<uint8_t>(n * 64);
        d_L2 = mem.alloc<uint8_t>(n * 128);
        d_aL = mem.alloc<uint8_t>(n * 64);
        d_bL = mem.alloc<uint8_t>(n * 64);
        const std::pair<const uint8_t*, uint8_t*> g1_sets[3] = {{d_tau1, d_L1}, {d_atau, d_aL}, {d_btau, d_bL}};
        for (const auto& s : g1_sets) {
            pts_from_affine_kernel<G1, Fq><<<pblocks, 128, 0, st>>>(s.first, (uint32_t)n, d_work);
            points_intt<G1, Fq>(dom, d_work, d_sc, s.second, st);
        }
        pts_from_affine_kernel<G2, Fq2><<<pblocks, 128, 0, st>>>(d_tau2, (uint32_t)n, d_work);
        points_intt<G2, Fq2>(dom, d_work, d_sc, d_L2, st);
        g_launch_count += 4;
    }

    // the H query
    uint8_t* d_h = mem.alloc<uint8_t>(n * 64);
    if (libsnark) {
        hq_libsnark_kernel<<<pblocks, 128, 0, st>>>(d_tau1, (uint32_t)n, d_h);
        g_launch_count += 1;
    } else if (lg) {
        // the odd entries of block log_n + 1, less the term of T_(2n-1) when that block is not the padded top one
        const uint8_t* d_blk = powers_upload(mem, "lagrange_tau_g1", (const uint8_t*)lg->tau_g1 + (2 * n - 1) * 64, 2 * n, false,
                                             false, st, 2 * n - 1);
        uint8_t* d_corr = nullptr;
        const uint8_t* last = (const uint8_t*)pw->tau_g1 + (2 * n - 1) * 64;
        if (logn < (int)lg->log_size && !all_zero(last, 64)) {
            const uint8_t* d_last = powers_upload(mem, "tau_g1", last, 1, false, false, st, 2 * n - 1);
            void* d_tab = mem.alloc<void>(32 * 255 * 64);
            fe* d_ks = mem.alloc<fe>(n * sizeof(fe));
            d_corr = mem.alloc<uint8_t>(n * 64);
            fixed_table_kernel<G1, Fq><<<(32 * 255 + 63) / 64, 64, 0, st>>>(d_tab, d_last);
            hq_lagrange_scalars_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((uint32_t)n, dom.tw, d_sc + 1, d_ks);
            fixed_base_kernel<G1, Fq><<<pblocks, 128, 0, st>>>(d_tab, d_ks, (uint32_t)n, d_corr);
            g_launch_count += 3;
        }
        hq_lagrange_kernel<<<pblocks, 128, 0, st>>>(d_blk, (uint32_t)n, d_corr, d_h);
        g_launch_count += 1;
    } else {
        hq_circom_kernel<<<pblocks, 128, 0, st>>>(d_tau1, (uint32_t)n, dom.tw, d_work);
        g_launch_count += 1;
        points_intt<G1, Fq>(dom, d_work, d_sc + 1, d_h, st);
    }
    CUDA_CHECK(cudaGetLastError());

    // column sums: a = A L, b1 = B L, b2 = B L2, k = A beta L + B alpha L + C L, then the public-input rows and affine form
    const ColPlan plans[3] = {col_plan(mem, d, 0, nv, st), col_plan(mem, d, 1, nv, st), col_plan(mem, d, 2, nv, st)};
    size_t scratch = 1;
    for (const ColPlan& cp : plans) if (cp.nnz) scratch = std::max(scratch, (size_t)cp.pieces[1]);
    uint8_t* d_x = mem.alloc<uint8_t>(scratch * 256);
    uint8_t* d_y = mem.alloc<uint8_t>(scratch * 256);
    uint8_t* d_acc = mem.alloc<uint8_t>((size_t)nv * (128 * 3 + 256));
    CUDA_CHECK(cudaMemsetAsync(d_acc, 0, (size_t)nv * (128 * 3 + 256), st));
    uint8_t *acc_a = d_acc, *acc_b1 = acc_a + (size_t)nv * 128, *acc_k = acc_b1 + (size_t)nv * 128, *acc_b2 = acc_k + (size_t)nv * 128;
    col_sums<G1, Fq>(plans[0], nv, m, d_L1, d_x, d_y, acc_a, st);
    col_sums<G1, Fq>(plans[1], nv, m, d_L1, d_x, d_y, acc_b1, st);
    col_sums<G2, Fq2>(plans[1], nv, m, d_L2, d_x, d_y, acc_b2, st);
    col_sums<G1, Fq>(plans[0], nv, m, d_bL, d_x, d_y, acc_k, st);
    col_sums<G1, Fq>(plans[1], nv, m, d_aL, d_x, d_y, acc_k, st);
    col_sums<G1, Fq>(plans[2], nv, m, d_L1, d_x, d_y, acc_k, st);
    uint8_t* d_out = mem.alloc<uint8_t>((size_t)nv * (64 * 3 + 128));
    uint8_t *out_a = d_out, *out_b1 = out_a + (size_t)nv * 64, *out_k = out_b1 + (size_t)nv * 64, *out_b2 = out_k + (size_t)nv * 64;
    const unsigned vblocks = (nv + 127) / 128;
    colsum_finish_kernel<G1, Fq><<<vblocks, 128, 0, st>>>(nv, ni, m, acc_a, d_L1, out_a);
    colsum_finish_kernel<G1, Fq><<<vblocks, 128, 0, st>>>(nv, ni, m, acc_b1, nullptr, out_b1);
    colsum_finish_kernel<G1, Fq><<<vblocks, 128, 0, st>>>(nv, ni, m, acc_k, d_bL, out_k);
    colsum_finish_kernel<G2, Fq2><<<vblocks, 128, 0, st>>>(nv, ni, m, acc_b2, nullptr, out_b2);
    g_launch_count += 4;
    CUDA_CHECK(cudaGetLastError());

    CUDA_CHECK(cudaMemcpyAsync(o->a_query, out_a, (size_t)nv * 64, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(o->b_g1_query, out_b1, (size_t)nv * 64, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(o->b_g2_query, out_b2, (size_t)nv * 128, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(o->gamma_abc_g1, out_k, (size_t)ni * 64, cudaMemcpyDeviceToHost, st));
    if (nv > ni) CUDA_CHECK(cudaMemcpyAsync(o->l_query, out_k + (size_t)ni * 64, (size_t)(nv - ni) * 64, cudaMemcpyDeviceToHost, st));
    if (nh) CUDA_CHECK(cudaMemcpyAsync(o->h_query, d_h, nh * 64, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    memcpy(o->alpha_g1, pw->alpha_tau_g1, 64);
    memcpy(o->beta_g1, pw->beta_tau_g1, 64);
    memcpy(o->delta_g1, pw->tau_g1, 64);
    memcpy(o->beta_g2, pw->beta_g2, 128);
    memcpy(o->gamma_g2, pw->tau_g2, 128);
    memcpy(o->delta_g2, pw->tau_g2, 128);
}

// b2g_points_intt: n = 2^logn affine points in place (host buffer)
static void points_intt_run(b2g_ctx* ctx, int g2, int logn, void* pts) {
    if (!ctx || !pts) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    if (logn < 1 || logn > 27) throw_error(B2G_E_DOMAIN, "b2g_points_intt: log_n must be in 1..27");
    const size_t n = (size_t)1 << logn, row = g2 ? 128 : 64;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st, true);
    uint8_t* d_in = mem.alloc<uint8_t>(n * row);
    uint8_t* d_work = mem.alloc<uint8_t>(n * row * 2);
    fe* d_sc = mem.alloc<fe>(2 * sizeof(fe));
    NttDomainHold dom(logn, st);
    pts_scale_kernel<<<1, 1, 0, st>>>(dom.ct, d_sc);
    g_launch_count += 2;
    CUDA_CHECK(cudaMemcpyAsync(d_in, pts, n * row, cudaMemcpyHostToDevice, st));
    const unsigned blocks = (unsigned)((n + 127) / 128);
    if (g2) {
        pts_from_affine_kernel<G2, Fq2><<<blocks, 128, 0, st>>>(d_in, (uint32_t)n, d_work);
        points_intt<G2, Fq2>(dom, d_work, d_sc, d_in, st);
    } else {
        pts_from_affine_kernel<G1, Fq><<<blocks, 128, 0, st>>>(d_in, (uint32_t)n, d_work);
        points_intt<G1, Fq>(dom, d_work, d_sc, d_in, st);
    }
    CUDA_CHECK(cudaMemcpyAsync(pts, d_in, n * row, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

// ---------------------------------------------------------------------------------------------- phase-2 preparation
constexpr int SEG_LOG = 16;                     // blocks of fewer than 2^SEG_LOG points run in the segmented pass
constexpr size_t PREP_PINNED = (size_t)64 << 20;  // bytes of the pinned buffer the output goes back through

// the sections of one curve in the segmented pass (grid.y picks one): per section its input (affine), how many input points
// there are (infinity beyond), its top block and its XYZZ work area and affine output, each block k at offset 2^k - 1
struct SegSet {
    const void* in[3];
    uint64_t limit[3];
    int top[3];
    void* work[3];
    void* out[3];
};

// work[2^k - 1 + i] = in[i] (infinity for i >= limit), k <= top, one point per thread
template <class C, class F>
__global__ void __launch_bounds__(128) seg_fill_kernel(SegSet s) {
    const int y = blockIdx.y;
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (2ull << s.top[y]) - 1) return;
    const uint64_t i = g + 1 - (1ull << (63 - __clzll(g + 1)));
    pt_store<F>(s.work[y], g, i < s.limit[y] ? C::from_affine(aff_load<F>(s.in[y], i)) : C::infinity());
}

// round t of the segmented transform: stage k - 1 - t (pts_intt_stage_kernel's butterfly) of every block k in t + 1 .. top.
// Block k has 2^(k-1) butterflies, so butterfly g of the round belongs to the block with 2^(k-1) <= g + 2^t < 2^k.  Its twiddle
// omega_(2^(k+1))^x is tw[x 2^(L-k)] in the table of a domain of 2^L >= 2^k points.
template <class C, class F>
__global__ void __launch_bounds__(128) seg_stage_kernel(SegSet s, int t, int L, const fe* __restrict__ tw) {
    const int y = blockIdx.y, top = s.top[y];
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (top <= t || g >= (1ull << top) - (1ull << t)) return;
    const uint64_t gg = g + (1ull << t);
    const int k = 64 - __clzll(gg), sg = k - 1 - t;
    const uint32_t b = (uint32_t)(gg - (1ull << (k - 1)));
    const uint32_t h = 1u << sg, j = b & (h - 1), i0 = ((b >> sg) << (sg + 1)) | j, i1 = i0 + h;
    const uint32_t e = j << t;
    void* pts = s.work[y];
    const uint64_t a0 = (1ull << k) - 1 + i0, a1 = (1ull << k) - 1 + i1;
    const typename C::Pt u = pt_load<F>(pts, a0);
    typename C::Pt v = pt_load<F>(pts, a1), sum = u;
    C::add(sum, v);
    C::add(v, C::neg(u));                                                  // v - u
    if (e) {
        const fe w = Fr::to_canonical(fe_load_nc(&tw[(size_t)((1u << k) - 2 * e) << (L - k)]));
        v = C::mul_scalar(v, w.l);
    } else {
        v = C::neg(v);
    }
    pt_store<F>(pts, a0, sum);
    pt_store<F>(pts, a1, v);
}

// out[2^k - 1 + i] = 2^-k work[2^k - 1 + bitrev_k(i)] in affine form, k <= top: every block's finish in one launch
template <class C, class F>
__global__ void __launch_bounds__(128) seg_finish_kernel(SegSet s, const fe* __restrict__ sc) {
    const int y = blockIdx.y;
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (2ull << s.top[y]) - 1) return;
    const int k = 63 - __clzll(g + 1);
    const uint32_t i = (uint32_t)(g + 1 - (1ull << k)), src = k ? __brev(i) >> (32 - k) : 0u;
    const fe scale = sc[k];
    aff_store<F>(s.out[y], g, C::to_affine(C::mul_scalar(pt_load<F>(s.work[y], ((1ull << k) - 1) + src), scale.l)));
}

// sc[k] = 2^-k (canonical), k < 28
__global__ void inv_pow2_kernel(fe* __restrict__ sc) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe two = fe_zero(); two.l[0] = 2;
    const fe half = Fr::inv(Fr::from_canonical(two));
    fe p = Fr::one();
    for (int k = 0; k < 28; k++) { sc[k] = Fr::to_canonical(p); p = Fr::mul(p, half); }
}

// host[0 .. bytes) = d[0 .. bytes) through the pinned buffer (host may be a memory-mapped file)
static void to_host(PinnedHost& pin, const uint8_t* d, size_t bytes, void* host, cudaStream_t st) {
    for (size_t off = 0; off < bytes; off += pin.bytes) {
        const size_t c = std::min(pin.bytes, bytes - off);
        CUDA_CHECK(cudaMemcpyAsync(pin.p, d + off, c, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        memcpy((uint8_t*)host + off, pin.p, c);
    }
}

static void powers_prepare_run(b2g_ctx* ctx, const b2g_powers_desc* pw, const b2g_lagrange_out* o) {
    if (!ctx || !pw || !o) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    if (pw->log_size > 28) throw_error(B2G_E_DOMAIN, "b2g_powers_prepare: log_size " + std::to_string(pw->log_size) + " exceeds 28");
    const int K = (int)o->log_size;
    if (K < 1 || K > 26 || K > (int)pw->log_size)
        throw_error(B2G_E_DOMAIN, "b2g_powers_prepare: power " + std::to_string(K) + " is outside 1.." +
                                      std::to_string(std::min<uint32_t>(pw->log_size, 26)));
    powers_arrays(pw, false);
    if (!o->tau_g1 || !o->tau_g2 || !o->alpha_tau_g1 || !o->beta_tau_g1) throw_error(B2G_E_SHAPE, "null output array");
    powers_first_finite(pw);
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st, true);
    const uint64_t nK = 1ull << K;
    // sections in launch order: the three G1 ones (one segmented launch), then G2
    struct Sec { const char* name; const uint8_t* in; uint8_t* out; uint64_t limit; int top; bool g2; };
    const Sec secs[4] = {{"tau_g1", (const uint8_t*)pw->tau_g1, (uint8_t*)o->tau_g1, 2 * nK - 1, K + 1, false},
                         {"alpha_tau_g1", (const uint8_t*)pw->alpha_tau_g1, (uint8_t*)o->alpha_tau_g1, nK, K, false},
                         {"beta_tau_g1", (const uint8_t*)pw->beta_tau_g1, (uint8_t*)o->beta_tau_g1, nK, K, false},
                         {"tau_g2", (const uint8_t*)pw->tau_g2, (uint8_t*)o->tau_g2, nK, K, true}};
    fe* d_sc = mem.alloc<fe>(28 * sizeof(fe));
    inv_pow2_kernel<<<1, 1, 0, st>>>(d_sc);
    g_launch_count += 1;
    PinnedHost pin(std::min(PREP_PINNED, (size_t)(4 * nK - 1) * 64));

    // blocks 0 .. min(top, SEG_LOG - 1) of every section: one segmented pass per curve
    SegSet set[2] = {};
    int seg_top = 0;
    for (int x = 0; x < 4; x++) {
        const Sec& c = secs[x];
        const int top = std::min(c.top, SEG_LOG - 1);
        const uint64_t cnt = std::min<uint64_t>(c.limit, 1ull << top), recs = (2ull << top) - 1;
        SegSet& s = set[c.g2 ? 1 : 0];
        const int y = c.g2 ? 0 : x;
        s.in[y] = powers_upload(mem, c.name, c.in, cnt, c.g2, c.g2, st);
        s.limit[y] = cnt;
        s.top[y] = top;
        s.work[y] = mem.alloc<uint8_t>(recs * (c.g2 ? 256 : 128));
        s.out[y] = mem.alloc<uint8_t>(recs * (c.g2 ? 128 : 64));
        seg_top = std::max(seg_top, top);
    }
    {
        NttDomainHold seg_dom(seg_top, st);
        const unsigned fill_blocks = (unsigned)(((2ull << seg_top) - 1 + 127) / 128);
        seg_fill_kernel<G1, Fq><<<dim3(fill_blocks, 3), 128, 0, st>>>(set[0]);
        seg_fill_kernel<G2, Fq2><<<dim3(fill_blocks, 1), 128, 0, st>>>(set[1]);
        g_launch_count += 2;
        const unsigned stage_blocks = (unsigned)(((1ull << seg_top) + 127) / 128);
        for (int t = 0; t < seg_top; t++) {
            seg_stage_kernel<G1, Fq><<<dim3(stage_blocks, 3), 128, 0, st>>>(set[0], t, seg_top, seg_dom.tw);
            seg_stage_kernel<G2, Fq2><<<dim3(stage_blocks, 1), 128, 0, st>>>(set[1], t, seg_top, seg_dom.tw);
        }
        seg_finish_kernel<G1, Fq><<<dim3(fill_blocks, 3), 128, 0, st>>>(set[0], d_sc);
        seg_finish_kernel<G2, Fq2><<<dim3(fill_blocks, 1), 128, 0, st>>>(set[1], d_sc);
        g_launch_count += 2 * seg_top + 2;
        CUDA_CHECK(cudaGetLastError());
        for (int x = 0; x < 4; x++) {
            const Sec& c = secs[x];
            const SegSet& s = set[c.g2 ? 1 : 0];
            const int y = c.g2 ? 0 : x;
            to_host(pin, (const uint8_t*)s.out[y], ((2ull << s.top[y]) - 1) * (c.g2 ? 128 : 64), c.out, st);
        }
    }

    // the larger blocks, one transform each, largest first, through one work area sized for the top block
    if (K + 1 < SEG_LOG) return;
    uint8_t* d_work = mem.alloc<uint8_t>((2 * nK) * 128);
    uint8_t* d_aff = mem.alloc<uint8_t>((2 * nK) * 64);
    for (const Sec& c : secs) {
        const size_t row = c.g2 ? 128 : 64;
        for (int k = c.top; k >= SEG_LOG; k--) {
            const uint64_t n = 1ull << k, cnt = std::min<uint64_t>(c.limit, n);
            check_upload(c.name, 0, c.in, cnt, c.g2, c.g2, d_aff, st);
            if (cnt < n) CUDA_CHECK(cudaMemsetAsync(d_aff + cnt * row, 0, (n - cnt) * row, st));
            NttDomainHold dom(k, st);
            const unsigned blocks = (unsigned)((n + 127) / 128);
            if (c.g2) {
                pts_from_affine_kernel<G2, Fq2><<<blocks, 128, 0, st>>>(d_aff, (uint32_t)n, d_work);
                points_intt<G2, Fq2>(dom, d_work, d_sc + k, d_aff, st);
            } else {
                pts_from_affine_kernel<G1, Fq><<<blocks, 128, 0, st>>>(d_aff, (uint32_t)n, d_work);
                points_intt<G1, Fq>(dom, d_work, d_sc + k, d_aff, st);
            }
            g_launch_count += 1;
            to_host(pin, d_aff, n * row, c.out + (n - 1) * row, st);
        }
    }
}

// ---------------------------------------------------------------------------------------------- delta contributions
// k[1] = x^-1 (canonical) from k[0] = x (canonical, nonzero, below r)
__global__ void delta_inverse_kernel(fe* __restrict__ k) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    k[1] = Fr::to_canonical(Fr::inv(Fr::from_canonical(k[0])));
}

// out[i] = k pts[i] (affine), one point per thread
template <class C, class F>
__global__ void __launch_bounds__(128) pts_scale_by_kernel(const void* __restrict__ pts, uint32_t n, const fe* __restrict__ k,
                                                           void* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fe s = *k;
    aff_store<F>(out, i, C::to_affine(aff_mul<C>(aff_load<F>(pts, i), s.l)));
}

static void delta_update_run(b2g_ctx* ctx, const b2g_delta_key* a, const void* x_canon, b2g_delta_key* b) {
    if (!ctx || !a || !x_canon || !b) throw_error(B2G_E_SHAPE, "null pointer");
    if (!a->delta_g1 || !a->delta_g2 || !b->delta_g1 || !b->delta_g2 || (a->n_l && (!a->l_query || !b->l_query)) ||
        (a->n_h && (!a->h_query || !b->h_query)))
        throw_error(B2G_E_SHAPE, "null key buffer");
    if (a->n_l != b->n_l || a->n_h != b->n_h) throw_error(B2G_E_SHAPE, "b2g_delta_update: the two keys' n_l / n_h differ");
    const CtxView cv = ctx_idle(ctx);
    if (!below((const uint8_t*)x_canon, R_WORDS)) throw_error(B2G_E_INPUT, "x is not below r");
    if (all_zero(x_canon, 32)) throw_error(B2G_E_INPUT, "x is zero");
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st, true);
    uint8_t* d_d1 = powers_upload(mem, "delta_g1", a->delta_g1, 1, false, false, st);
    uint8_t* d_d2 = powers_upload(mem, "delta_g2", a->delta_g2, 1, true, true, st);
    uint8_t* d_l = powers_upload(mem, "l_query", a->l_query, a->n_l, false, false, st);
    uint8_t* d_h = powers_upload(mem, "h_query", a->h_query, a->n_h, false, false, st);
    fe* d_k = mem.alloc<fe>(2 * sizeof(fe));
    upload_secrets(d_k, &x_canon, 1, st);
    delta_inverse_kernel<<<1, 1, 0, st>>>(d_k);
    const size_t most = std::max((size_t)std::max(a->n_l, a->n_h), (size_t)2);
    uint8_t* d_out = mem.alloc<uint8_t>(most * 64);
    uint8_t* d_out2 = mem.alloc<uint8_t>(128);
    pts_scale_by_kernel<G1, Fq><<<1, 128, 0, st>>>(d_d1, 1, d_k, d_out);
    pts_scale_by_kernel<G2, Fq2><<<1, 128, 0, st>>>(d_d2, 1, d_k, d_out2);
    g_launch_count += 3;
    CUDA_CHECK(cudaMemcpyAsync(b->delta_g1, d_out, 64, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(b->delta_g2, d_out2, 128, cudaMemcpyDeviceToHost, st));
    const std::pair<const uint8_t*, std::pair<uint32_t, void*>> qs[2] = {{d_l, {a->n_l, b->l_query}}, {d_h, {a->n_h, b->h_query}}};
    for (const auto& q : qs) {
        const uint32_t n = q.second.first;
        if (!n) continue;
        CUDA_CHECK(cudaStreamSynchronize(st));                             // d_out is reused
        pts_scale_by_kernel<G1, Fq><<<(n + 127) / 128, 128, 0, st>>>(q.first, n, d_k + 1, d_out);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(q.second.second, d_out, (size_t)n * 64, cudaMemcpyDeviceToHost, st));
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(st));
}

}  // namespace b2g

extern "C" {

int b2g_setup(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_setup_secrets* secrets, b2g_setup_out* out) {
    return b2g::guarded_clear([&] { b2g::setup_run(ctx, circuit, secrets, out); });
}

int b2g_setup_from_powers(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers, b2g_setup_out* out) {
    return b2g::guarded_clear([&] { b2g::setup_from_powers_run(ctx, circuit, powers, out); });
}

int b2g_points_intt(b2g_ctx* ctx, int g2, int log_n, void* points_mont) {
    return b2g::guarded_clear([&] { b2g::points_intt_run(ctx, g2, log_n, points_mont); });
}

int b2g_setup_from_lagrange(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers, const b2g_lagrange_desc* lagrange,
                            b2g_setup_out* out) {
    return b2g::guarded_clear([&] {
        if (!lagrange) b2g::throw_error(B2G_E_SHAPE, "null pointer");
        b2g::setup_from_powers_run(ctx, circuit, powers, out, lagrange);
    });
}

int b2g_powers_prepare(b2g_ctx* ctx, const b2g_powers_desc* powers, const b2g_lagrange_out* out) {
    return b2g::guarded_clear([&] { b2g::powers_prepare_run(ctx, powers, out); });
}

int b2g_delta_update(b2g_ctx* ctx, const b2g_delta_key* before, const void* x_canon, b2g_delta_key* after) {
    return b2g::guarded_clear([&] { b2g::delta_update_run(ctx, before, x_canon, after); });
}

}  // extern "C"
