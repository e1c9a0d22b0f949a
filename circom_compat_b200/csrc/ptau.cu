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
//
// b2g_setup_check, a proving key against its circuit and ceremony, moves b2g_setup_from_powers's point transforms onto scalars:
//   weights       w_j = rho^j and v_i = sigma^i by the powers kernels of the streamed MSM
//   row products  c = A'w, Bw, Cw: one product per nonzero keyed by its row, then a reduce-by-key with the Fr addition, so a
//                 row holding every column is summed by many threads; the public-input rows of A' add w_j at row m + j
//   transforms    s = iNTT_n(c) on the scalar NTT; the E5 scalars h from v by the reduction's formula
//   sums          the same streamed passes as above: the key's arrays with the powers of rho (sigma for h_query), the ceremony's
//                 with the explicit scalars s and h; the point rules (setup_rules, verify.cu) in the same passes
//   verdict       setup_check_verdict_kernel (verify.cu): E1-E3 compare sums, E4-E6 are three pairing products
// Every scalar is canonical: the Montgomery product of a Montgomery coefficient and a canonical weight is the canonical product,
// and the transform, being linear, maps canonical inputs to canonical outputs.
#include <algorithm>
#include <cstring>
#include <string>
#include "../../include/b2groth.h"
#include "msm.cuh"
#include "ntt.cuh"
#include "setup.cuh"
#include "stage.cuh"
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

__global__ void to_mont_kernel(const fe* __restrict__ canon, uint32_t n, fe* __restrict__ mont) {
    if (threadIdx.x == 0 && blockIdx.x == 0)
        for (uint32_t j = 0; j < n; j++) mont[j] = Fr::from_canonical(canon[j]);
}

void to_mont(const fe* canon, uint32_t n, fe* mont, cudaStream_t st) {
    to_mont_kernel<<<1, 1, 0, st>>>(canon, n, mont);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

template <class C, class F>
__global__ void powers_affine_kernel(const void* __restrict__ acc, void* __restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) aff_store<F>(out, 0, C::to_affine(pt_load<F>(acc, 0)));
}

struct MsmHold {
    PowersMsm m;
    cudaStream_t st;
    MsmHold(bool g2, uint64_t count, cudaStream_t s) : st(s) { powers_msm_alloc(m, g2, (uint32_t)std::min<uint64_t>(count, POWERS_SLICE)); }
    ~MsmHold() { cudaStreamSynchronize(st); powers_msm_free(m); }
};

// one pass over `count` host points: with bad, the point rules (b2g_powers_check's, gen: point 0 must be the generator; with
// loose, b2g_setup_check's); with msm, msm->acc = sum_i k_i X_i, k_i = rho^(start + i) or, with scalars (device), scalars[i]
static void powers_pass(Staging& sg, PowersMsm* msm, bool g2, const void* host, uint64_t count, bool gen, unsigned long long* bad,
                        const fe* rho, bool loose = false, uint64_t start = 0, const fe* scalars = nullptr) {
    const size_t row = g2 ? 128 : 64;
    if (msm) powers_msm_reset(*msm, sg.st);
    uint64_t k = 0;
    for (uint64_t off = 0; off < count; off += POWERS_SLICE, k++) {
        const uint32_t cnt = (uint32_t)std::min<uint64_t>(POWERS_SLICE, count - off);
        const int b = (int)(k & 1);
        const uint8_t* d = sg.upload(b, (const uint8_t*)host + off * row, (size_t)cnt * row);
        if (bad && loose) setup_rules(g2, d, cnt, off, bad, sg.st);
        else if (bad) powers_rules(g2, d, cnt, off, gen, bad, sg.st);
        if (msm) powers_msm_slice(*msm, d, cnt, start + off, rho, sg.st, scalars ? scalars + off : nullptr);
        CUDA_CHECK(cudaEventRecord(sg.used[b], sg.st));
    }
}

static void powers_msm_run(b2g_ctx* ctx, int g2, size_t n, const void* bases, const void* rho, void* out) {
    if (!ctx || !rho || !out || (n && !bases)) throw_error(B2G_E_SHAPE, "null pointer");
    const CtxView cv = ctx_idle(ctx);
    const uint8_t* r = (const uint8_t*)rho;
    if (!below(r, R_WORDS)) throw_error(B2G_E_INPUT, "rho is not below r");
    const size_t row = g2 ? 128 : 64;
    if (n == 0) { memset(out, 0, row); return; }
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st);
    uint8_t* V = mem.alloc(PV_BYTES);
    MsmHold h(g2 != 0, n, st);
    Staging sg(std::min<size_t>(n, POWERS_SLICE) * row, st);
    fe* d_rho = (fe*)(V + PV_RHO);
    CUDA_CHECK(cudaMemcpyAsync(V + PV_CH, rho, 32, cudaMemcpyHostToDevice, st));
    to_mont((const fe*)(V + PV_CH), 1, d_rho, st);
    powers_pass(sg, &h.m, g2 != 0, bases, n, false, nullptr, d_rho);
    if (g2) powers_affine_kernel<G2, Fq2><<<1, 1, 0, st>>>(h.m.acc, V + PV_POINT);
    else powers_affine_kernel<G1, Fq><<<1, 1, 0, st>>>(h.m.acc, V + PV_POINT);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, V + PV_POINT, row, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

static void powers_check_run(b2g_ctx* ctx, const b2g_powers_desc* pw, uint32_t log_n, const void* challenges, b2g_powers_report* out) {
    if (!ctx || !pw || !challenges || !out) throw_error(B2G_E_SHAPE, "null pointer");
    memset(out, 0, sizeof(*out));
    const CtxView cv = ctx_idle(ctx);
    if (pw->log_size > 28) throw_error(B2G_E_DOMAIN, "b2g_powers_check: log_size " + std::to_string(pw->log_size) + " exceeds 28");
    if (log_n < 1 || log_n > pw->log_size)
        throw_error(B2G_E_DOMAIN, "b2g_powers_check: log_n " + std::to_string(log_n) + " is outside 1.." + std::to_string(pw->log_size));
    powers_arrays(pw, true);
    static const char* const CH_NAMES[5] = {"rho", "sigma", "pi", "kappa", "eps"};
    for (int k = 0; k < 5; k++)
        if (!scalar_ok((const uint8_t*)challenges + 32 * k)) throw_error(B2G_E_INPUT, std::string("challenge ") + CH_NAMES[k] + " is 0 or >= r");
    const uint64_t n = 1ull << log_n;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st);
    uint8_t* V = mem.alloc(PV_BYTES);
    MsmHold h1(false, 2 * n - 1, st), h2(true, n, st);
    Staging sg(std::max<size_t>(std::min<uint64_t>(2 * n - 1, POWERS_SLICE) * 64, std::min<uint64_t>(n, POWERS_SLICE) * 128), st);
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
    to_mont((const fe*)(V + PV_CH), 1, (fe*)(V + PV_RHO), st);

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
        const uint32_t rule = bad_point_rule("b2g_powers_check", x.host, bad, x.g2, x.gen, V + PV_POINT, (uint32_t*)(V + PV_WORD), st);
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

// ---------------------------------------------------------------------------------------------- b2g_setup_check
// mont[0] = rho, mont[1] = sigma, mont[2] = 1/2 (Montgomery) from canon = rho, sigma
__global__ void check_consts_kernel(const fe* __restrict__ canon, fe* __restrict__ mont) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe two = fe_zero(); two.l[0] = 2;
    mont[0] = Fr::from_canonical(canon[0]);
    mont[1] = Fr::from_canonical(canon[1]);
    mont[2] = Fr::inv(Fr::from_canonical(two));
}

// prod[k] = val[k] w[col[k]] (canonical) and row[k] = the row of nonzero k
__global__ void __launch_bounds__(256) check_products_kernel(uint32_t nnz, uint32_t m, const uint32_t* __restrict__ rowptr,
                                                             const uint32_t* __restrict__ col, const fe* __restrict__ val,
                                                             const fe* __restrict__ w, fe* __restrict__ prod, uint32_t* __restrict__ row) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nnz) return;
    const uint32_t r = mat_row(rowptr, m, k);
    fe_store(&prod[k], Fr::mul(fe_load_nc(&val[k]), fe_load_nc(&w[col[k]])));
    row[k] = r;
}

// the public-input rows of A': c[m + j] = w[j], j < ni
__global__ void __launch_bounds__(256) check_public_rows_kernel(uint32_t ni, uint32_t m, const fe* __restrict__ w, fe* __restrict__ c) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < ni) fe_store(&c[m + j], fe_load(&w[j]));
}

// E5's scalars h (2n - 1, canonical).  CircomReduction: t = iNTT_n(v) at v, h_k = t_k omega_2n^-k / 2 and h_(k+n) = -h_k with
// omega_2n^-k = -tw[n - k] for k > 0; LibsnarkReduction: v = sigma^i, h_k = -v_k (k < n - 1), h_(n-1) = 0, h_(k+n) = v_k
__global__ void __launch_bounds__(256) check_h_kernel(uint32_t n, int libsnark, const fe* __restrict__ v, const fe* __restrict__ tw,
                                                      const fe* __restrict__ half, fe* __restrict__ h) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    fe lo, hi;
    if (libsnark) {
        hi = fe_load(&v[k]);
        lo = k + 1 < n ? Fr::neg(hi) : fe_zero();
    } else {
        lo = Fr::mul(fe_load(&v[k]), *half);
        if (k) lo = Fr::neg(Fr::mul(lo, fe_load_nc(&tw[n - k])));
        hi = Fr::neg(lo);
    }
    fe_store(&h[k], lo);
    if (k + 1 < n) fe_store(&h[n + k], hi);
}

static const char* const KEY_NAMES[12] = {"alpha_g1", "beta_g1", "delta_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1", "a_query",
                                          "b_g1_query", "b_g2_query", "l_query", "h_query"};

// the small device buffer of a key check: its layout
enum : size_t {
    SK_SUMS = 0,                     // the SC_ records (verify.cuh)
    SK_G1 = SC_BYTES,                // delta_1, T_0 (affine)
    SK_G2 = SK_G1 + 2 * 64,          // gamma_2, delta_2, U_0 (affine)
    SK_CH = SK_G2 + 3 * 128,         // rho, sigma (canonical)
    SK_MONT = SK_CH + 2 * 32,        // rho, sigma, 1/2 (Montgomery)
    SK_PW = SK_MONT + 3 * 32,        // the powers kernels' two words
    SK_BAD = SK_PW + 2 * 32,         // the lowest failing index of the 5 ceremony arrays, then of the 12 key fields
    SK_POINT = SK_BAD + 160,         // the point a failure names (128 B)
    SK_WORD = SK_POINT + 128,        // the verdict, or the failing point's rule
    SK_RUNS = SK_WORD + 4,
    SK_BYTES = SK_RUNS + 4
};

static void setup_check_run(b2g_ctx* ctx, const b2g_mat_desc* d, const b2g_powers_desc* pw, const b2g_key_desc* key, const void* challenges,
                            b2g_setup_report* out) {
    if (!ctx || !d || !pw || !key || !challenges || !out) throw_error(B2G_E_SHAPE, "null pointer");
    memset(out, 0, sizeof(*out));
    const CtxView cv = ctx_idle(ctx);
    const int logn = setup_domain(d);
    const bool libsnark = d->reduction == B2G_REDUCTION_LIBSNARK;
    powers_cover(pw, logn);
    powers_arrays(pw, true);
    static const char* const CH_NAMES[2] = {"rho", "sigma"};
    for (int k = 0; k < 2; k++)
        if (!scalar_ok((const uint8_t*)challenges + 32 * k)) throw_error(B2G_E_INPUT, std::string("challenge ") + CH_NAMES[k] + " is 0 or >= r");
    const void* fields[12] = {key->alpha_g1, key->beta_g1, key->delta_g1, key->beta_g2, key->gamma_g2, key->delta_g2,
                              key->gamma_abc_g1, key->a_query, key->b_g1_query, key->b_g2_query, key->l_query, key->h_query};
    const uint64_t counts[12] = {1, 1, 1, 1, 1, 1, key->n_ic, key->n_vars, key->n_vars, key->n_vars, key->n_l, key->n_h};
    for (int f = 0; f < 12; f++)
        if (counts[f] && !fields[f]) throw_error(B2G_E_SHAPE, std::string("null key field ") + KEY_NAMES[f]);
    const uint32_t m = d->num_constraints, ni = d->num_inputs, nv = d->n_vars;
    const uint32_t maxnnz = max_nnz(d, "b2g_setup_check");
    const uint32_t n = 1u << logn, nh = libsnark ? n - 1 : n;
    out->ok = 0;

    // the counts, then the fields snarkjs copies from the ceremony
    const std::pair<uint32_t, uint32_t> shapes[4] = {{7, nv}, {6, ni}, {10, nv - ni}, {11, nh}};
    const uint32_t have[4] = {key->n_vars, key->n_ic, key->n_l, key->n_h};
    for (int k = 0; k < 4; k++)
        if (have[k] != shapes[k].second) { out->rule = 6; out->field = (uint8_t)shapes[k].first; out->index = shapes[k].second; return; }
    const std::pair<const void*, size_t> same[4] = {{pw->alpha_tau_g1, 64}, {pw->beta_tau_g1, 64}, {pw->beta_g2, 128}, {pw->tau_g2, 128}};
    const int same_field[4] = {0, 1, 3, 4};
    for (int k = 0; k < 4; k++)
        if (memcmp(fields[same_field[k]], same[k].first, same[k].second)) { out->rule = 7; out->field = (uint8_t)same_field[k]; return; }

    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st);
    uint8_t* V = mem.alloc(SK_BYTES);
    // the scalars: w (N), v then t (n), s^A, s^B, s^C (n each), h (2n; also the transforms' scratch before it holds h)
    fe* d_w = mem.alloc<fe>(((size_t)nv + 6 * (size_t)n) * sizeof(fe));
    fe *d_v = d_w + nv, *d_s[3] = {d_v + n, d_v + 2 * (size_t)n, d_v + 3 * (size_t)n}, *d_h = d_v + 4 * (size_t)n;
    fe* d_mont = (fe*)(V + SK_MONT);
    unsigned long long* d_bad = (unsigned long long*)(V + SK_BAD);
    CUDA_CHECK(cudaMemsetAsync(V, 0, SK_BYTES, st));
    CUDA_CHECK(cudaMemsetAsync(d_bad, 0xff, 17 * 8, st));
    CUDA_CHECK(cudaMemcpyAsync(V + SK_CH, challenges, 64, cudaMemcpyHostToDevice, st));
    check_consts_kernel<<<1, 1, 0, st>>>((const fe*)(V + SK_CH), d_mont);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
    powers_scalars(d_mont, 0, nv, (fe*)(V + SK_PW), d_w, st);
    powers_scalars(d_mont + 1, 0, n, (fe*)(V + SK_PW), d_v, st);

    // c = A'w, Bw, Cw by rows
    CUDA_CHECK(cudaMemsetAsync(d_s[0], 0, 3 * (size_t)n * sizeof(fe), st));
    if (maxnnz) {
        DevArena mat(st);                                              // freed at the end of this block
        uint32_t *rowptr = mat.alloc<uint32_t>(((size_t)m + 1) * 4), *col = mat.alloc<uint32_t>((size_t)maxnnz * 4);
        fe* val = mat.alloc<fe>((size_t)maxnnz * sizeof(fe));
        uint32_t *rows = mat.alloc<uint32_t>((size_t)maxnnz * 4), *uniq = mat.alloc<uint32_t>((size_t)maxnnz * 4);
        fe *prod = mat.alloc<fe>((size_t)maxnnz * sizeof(fe)), *agg = mat.alloc<fe>((size_t)maxnnz * sizeof(fe));
        uint32_t* d_runs = (uint32_t*)(V + SK_RUNS);
        size_t temp_bytes = 0;
        sum_by_key(nullptr, temp_bytes, rows, uniq, prod, agg, d_runs, maxnnz, nullptr, st);
        void* temp = mat.alloc<void>(temp_bytes);
        for (int x = 0; x < 3; x++) {
            const uint32_t nnz = mat_nnz(d, x);
            if (!nnz) continue;
            mat_upload(d, x, rowptr, col, val, st);
            check_products_kernel<<<(nnz + 255) / 256, 256, 0, st>>>(nnz, m, rowptr, col, val, d_w, prod, rows);
            g_launch_count += 1;
            size_t bytes = temp_bytes;
            sum_by_key(temp, bytes, rows, uniq, prod, agg, d_runs, nnz, d_s[x], st);
        }
    }
    check_public_rows_kernel<<<(ni + 255) / 256, 256, 0, st>>>(ni, m, d_w, d_s[0]);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // s = iNTT_n(c), in place; then h
    NttDomainHold dom(logn, st);
    for (int x = 0; x < 3; x++) ntt_plain(dom, d_s[x], d_h, true, st);
    if (!libsnark) ntt_plain(dom, d_v, d_h, true, st);
    check_h_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, libsnark ? 1 : 0, d_v, dom.tw, d_mont + 2, d_h);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());

    // the streamed passes: ceremony arrays (rules on the prefix b2g_setup_from_powers reads), then the key's fields
    const uint64_t g1_most = std::max<uint64_t>(2 * (uint64_t)n - 1, nv), g2_most = std::max<uint64_t>(n, nv);
    MsmHold h1(false, g1_most, st), h2(true, g2_most, st);
    Staging sg(std::max<size_t>(std::min<uint64_t>(g1_most, POWERS_SLICE) * 64, std::min<uint64_t>(g2_most, POWERS_SLICE) * 128), st);
    const void* T = pw->tau_g1;
    struct Pass { const void* host; uint64_t count; bool g2; int bad; const fe* rho; uint64_t start; const fe* scalars; size_t sum; };
    const fe *rho = d_mont, *sigma = d_mont + 1;
    const Pass passes[20] = {
        {T, 2 * (uint64_t)n - 1, false, 0, nullptr, 0, d_h, SC_RH}, {pw->tau_g2, n, true, 1, nullptr, 0, d_s[1], SC_RB2},
        {pw->alpha_tau_g1, n, false, 2, nullptr, 0, d_s[1], SC_RAL}, {pw->beta_tau_g1, n, false, 3, nullptr, 0, d_s[0], SC_RBE},
        {pw->beta_g2, 1, true, 4, nullptr, 0, nullptr, 0},
        {T, n, false, -1, nullptr, 0, d_s[0], SC_RA}, {T, n, false, -1, nullptr, 0, d_s[1], SC_RB1}, {T, n, false, -1, nullptr, 0, d_s[2], SC_RC},
        {fields[0], 1, false, 5, nullptr, 0, nullptr, 0}, {fields[1], 1, false, 6, nullptr, 0, nullptr, 0},
        {fields[2], 1, false, 7, nullptr, 0, nullptr, 0}, {fields[3], 1, true, 8, nullptr, 0, nullptr, 0},
        {fields[4], 1, true, 9, nullptr, 0, nullptr, 0}, {fields[5], 1, true, 10, nullptr, 0, nullptr, 0},
        {fields[6], ni, false, 11, rho, 0, nullptr, SC_KIC}, {fields[7], nv, false, 12, rho, 0, nullptr, SC_KA},
        {fields[8], nv, false, 13, rho, 0, nullptr, SC_KB1}, {fields[9], nv, true, 14, rho, 0, nullptr, SC_KB2},
        {fields[10], nv - ni, false, 15, rho, ni, nullptr, SC_KL}, {fields[11], nh, false, 16, sigma, 0, nullptr, SC_KH}};
    for (const Pass& p : passes) {
        const bool sum = p.rho || p.scalars;
        PowersMsm* msm = sum ? (p.g2 ? &h2.m : &h1.m) : nullptr;
        powers_pass(sg, msm, p.g2, p.host, p.count, false, p.bad >= 0 ? d_bad + p.bad : nullptr, p.rho, true, p.start, p.scalars);
        if (msm) CUDA_CHECK(cudaMemcpyAsync(V + SK_SUMS + p.sum, msm->acc, p.g2 ? 256 : 128, cudaMemcpyDeviceToDevice, st));
    }
    uint64_t bad[17];
    CUDA_CHECK(cudaMemcpyAsync(bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    // the points that must not be at infinity: tau_g1[0], tau_g2[0], delta_g1, delta_g2
    if (all_zero(T, 64)) bad[0] = 0;
    if (all_zero(pw->tau_g2, 128)) bad[1] = 0;
    if (all_zero(key->delta_g1, 64)) bad[7] = 0;
    if (all_zero(key->delta_g2, 128)) bad[10] = 0;
    // the first failing point in pass order, which is report order: the ceremony's arrays, then the key's fields
    for (const Pass& p : passes) {
        if (p.bad < 0 || bad[p.bad] >= p.count) continue;
        const uint32_t rule = bad_point_rule("b2g_setup_check", p.host, bad[p.bad], p.g2, false, V + SK_POINT, (uint32_t*)(V + SK_WORD), st);
        out->rule = (uint8_t)rule; out->side = p.bad < 5 ? 1 : 0; out->field = (uint8_t)(p.bad < 5 ? p.bad : p.bad - 5);
        out->index = bad[p.bad];
        return;
    }

    const std::pair<const void*, size_t> pts[5] = {{key->delta_g1, 64}, {T, 64}, {key->gamma_g2, 128}, {key->delta_g2, 128}, {pw->tau_g2, 128}};
    for (int k = 0, off = 0; k < 5; off += (int)pts[k].second, k++)
        CUDA_CHECK(cudaMemcpyAsync(V + SK_G1 + off, pts[k].first, pts[k].second, cudaMemcpyHostToDevice, st));
    setup_check_verdict(V + SK_SUMS, V + SK_G1, V + SK_G2, (uint32_t*)(V + SK_WORD), st);
    uint32_t verdict = 0;
    CUDA_CHECK(cudaMemcpyAsync(&verdict, V + SK_WORD, 4, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    static const uint8_t EQ_FIELD[7] = {0, 7, 8, 9, 6, 11, 2};
    if (verdict) { out->rule = 8; out->field = EQ_FIELD[verdict > 6 ? 0 : verdict]; return; }
    out->ok = 1;
}

// ---------------------------------------------------------------------------------------------- b2g_lagrange_check
// s[j] += t[j], j < n (canonical)
__global__ void __launch_bounds__(256) lagrange_accumulate_kernel(uint32_t n, const fe* __restrict__ t, fe* __restrict__ s) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) fe_store(&s[j], Fr::add(fe_load(&s[j]), fe_load(&t[j])));
}

// the small device buffer of a Lagrange check: its layout
enum : size_t {
    LC_AFF = 0,                      // the eight sums in affine form: per section the Lagrange side, then the monomial side
    LC_CH = LC_AFF + 2 * (3 * 64 + 128),
    LC_RHO = LC_CH + 32,             // rho (Montgomery)
    LC_PW = LC_RHO + 32,             // the powers kernels' two words
    LC_BAD = LC_PW + 64,             // the lowest failing index of each Lagrange section
    LC_POINT = LC_BAD + 4 * 8,
    LC_WORD = LC_POINT + 128,
    LC_BYTES = LC_WORD + 32
};

static void lagrange_check_run(b2g_ctx* ctx, const b2g_powers_desc* pw, const b2g_lagrange_desc* lg, uint32_t log_n, const void* rho,
                               b2g_powers_report* out) {
    if (!ctx || !pw || !lg || !rho || !out) throw_error(B2G_E_SHAPE, "null pointer");
    memset(out, 0, sizeof(*out));
    const CtxView cv = ctx_idle(ctx);
    const uint32_t p = lg->log_size;
    if (p > 26 || p > pw->log_size)
        throw_error(B2G_E_DOMAIN, "b2g_lagrange_check: Lagrange sections of power " + std::to_string(p) + " exceed 26 or the ceremony's power " +
                                      std::to_string(pw->log_size));
    if (log_n < 1 || log_n > p)
        throw_error(B2G_E_DOMAIN, "b2g_lagrange_check: log_n " + std::to_string(log_n) + " is outside 1.." + std::to_string(p));
    powers_arrays(pw, false);
    if (!lg->tau_g1 || !lg->tau_g2 || !lg->alpha_tau_g1 || !lg->beta_tau_g1) throw_error(B2G_E_SHAPE, "null Lagrange array");
    if (!scalar_ok((const uint8_t*)rho)) throw_error(B2G_E_INPUT, "challenge rho is 0 or >= r");
    const uint64_t n = 1ull << log_n;
    // section 12 reads blocks 0 .. log_n + 1 and 2n monomials, less the infinity that pads block p + 1
    const uint64_t n12 = 4 * n - 1, n13 = 2 * n - 1, t12 = log_n == p ? 2 * n - 1 : 2 * n;
    DevGuard g(cv.device);
    cudaStream_t st = cv.st;
    DevArena mem(st);
    uint8_t* V = mem.alloc(LC_BYTES);
    fe* d_rho = (fe*)(V + LC_RHO);
    unsigned long long* d_bad = (unsigned long long*)(V + LC_BAD);
    CUDA_CHECK(cudaMemsetAsync(V, 0, LC_BYTES, st));
    CUDA_CHECK(cudaMemsetAsync(d_bad, 0xff, 4 * 8, st));
    CUDA_CHECK(cudaMemcpyAsync(V + LC_CH, rho, 32, cudaMemcpyHostToDevice, st));
    to_mont((const fe*)(V + LC_CH), 1, d_rho, st);

    // the weights w_g = rho^g (g < 4n - 1), then s = sum_k pad(iNTT_(2^k)(w of block k)): s13 over blocks 0 .. log_n, s12 the
    // same plus block log_n + 1
    fe* d_w = mem.alloc<fe>((n12 + 4 * 2 * n) * sizeof(fe));       // w, then s12, s13, t and the transforms' scratch
    fe *d_s12 = d_w + n12, *d_s13 = d_s12 + 2 * n, *d_t = d_s13 + 2 * n, *d_tmp = d_t + 2 * n;
    powers_scalars(d_rho, 0, (uint32_t)n12, (fe*)(V + LC_PW), d_w, st);
    CUDA_CHECK(cudaMemsetAsync(d_s13, 0, 2 * n * sizeof(fe), st));
    for (uint32_t k = 0; k <= log_n + 1; k++) {
        const uint64_t m = 1ull << k;
        CUDA_CHECK(cudaMemcpyAsync(d_t, d_w + (m - 1), m * sizeof(fe), cudaMemcpyDeviceToDevice, st));
        if (k) {
            NttDomainHold dom((int)k, st);
            ntt_plain(dom, d_t, d_tmp, true, st);
            CUDA_CHECK(cudaStreamSynchronize(st));                     // dom is freed at the end of this block
        }
        if (k == log_n + 1) CUDA_CHECK(cudaMemcpyAsync(d_s12, d_s13, 2 * n * sizeof(fe), cudaMemcpyDeviceToDevice, st));
        lagrange_accumulate_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>((uint32_t)m, d_t, k == log_n + 1 ? d_s12 : d_s13);
        g_launch_count += 1;
        CUDA_CHECK(cudaGetLastError());
    }

    // the streamed passes: each Lagrange section with the powers of rho and its point rules, then its monomials with s
    MsmHold h1(false, n12, st), h2(true, n13, st);
    Staging sg(std::max<size_t>(std::min<uint64_t>(n12, POWERS_SLICE) * 64, std::min<uint64_t>(n13, POWERS_SLICE) * 128), st);
    struct Sec { const void* lag; uint64_t count; const void* mono; uint64_t terms; const fe* s; bool g2; };
    const Sec secs[4] = {{lg->tau_g1, n12, pw->tau_g1, t12, d_s12, false}, {lg->tau_g2, n13, pw->tau_g2, n, d_s13, true},
                         {lg->alpha_tau_g1, n13, pw->alpha_tau_g1, n, d_s13, false}, {lg->beta_tau_g1, n13, pw->beta_tau_g1, n, d_s13, false}};
    size_t off = LC_AFF;
    size_t at[4][2];
    for (int x = 0; x < 4; x++) {
        const Sec& c = secs[x];
        PowersMsm& msm = c.g2 ? h2.m : h1.m;
        const size_t row = c.g2 ? 128 : 64;
        for (int side = 0; side < 2; side++) {
            if (side == 0) powers_pass(sg, &msm, c.g2, c.lag, c.count, false, d_bad + x, d_rho, true);
            else powers_pass(sg, &msm, c.g2, c.mono, c.terms, false, nullptr, nullptr, false, 0, c.s);
            if (c.g2) powers_affine_kernel<G2, Fq2><<<1, 1, 0, st>>>(msm.acc, V + off);
            else powers_affine_kernel<G1, Fq><<<1, 1, 0, st>>>(msm.acc, V + off);
            g_launch_count += 1;
            CUDA_CHECK(cudaGetLastError());
            at[x][side] = off;
            off += row;
        }
    }
    uint8_t sums[LC_CH];
    uint64_t bad[4];
    CUDA_CHECK(cudaMemcpyAsync(sums, V, sizeof(sums), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaMemcpyAsync(bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    for (int x = 0; x < 4; x++) {
        const Sec& c = secs[x];
        if (bad[x] >= c.count) continue;
        const uint32_t rule = bad_point_rule("b2g_lagrange_check", c.lag, bad[x], c.g2, false, V + LC_POINT, (uint32_t*)(V + LC_WORD), st);
        out->rule = (uint8_t)rule; out->array = (uint8_t)(5 + x); out->index = bad[x];
        return;
    }
    for (int x = 0; x < 4; x++)
        if (memcmp(sums + at[x][0], sums + at[x][1], secs[x].g2 ? 128 : 64)) { out->rule = 7; out->array = (uint8_t)(5 + x); return; }
    out->ok = 1;
}

}  // namespace b2g

extern "C" {

int b2g_powers_msm(b2g_ctx* ctx, int g2, size_t n, const void* bases, const void* rho_canon, void* out_affine) {
    return b2g::guarded_clear([&] { b2g::powers_msm_run(ctx, g2, n, bases, rho_canon, out_affine); });
}

int b2g_powers_check(b2g_ctx* ctx, const b2g_powers_desc* powers, uint32_t log_n, const void* challenges, b2g_powers_report* out) {
    return b2g::guarded_clear([&] { b2g::powers_check_run(ctx, powers, log_n, challenges, out); });
}

int b2g_lagrange_check(b2g_ctx* ctx, const b2g_powers_desc* powers, const b2g_lagrange_desc* lagrange, uint32_t log_n,
                       const void* rho_canon, b2g_powers_report* out) {
    return b2g::guarded_clear([&] { b2g::lagrange_check_run(ctx, powers, lagrange, log_n, rho_canon, out); });
}

int b2g_setup_check(b2g_ctx* ctx, const b2g_mat_desc* circuit, const b2g_powers_desc* powers, const b2g_key_desc* key,
                    const void* challenges, b2g_setup_report* report) {
    return b2g::guarded_clear([&] { b2g::setup_check_run(ctx, circuit, powers, key, challenges, report); });
}

}  // extern "C"
