// ntt.cu - the R1CS -> QAP witness map of CircomReduction on the device.
//
// Replaces /root/reference/src/circom/qap.rs:23-88 (witness_map_from_matrices) and the ark-poly 0.5.0
// Radix2EvaluationDomain calls it makes (ifft_in_place / distribute_powers / fft_in_place / pointwise product).
// The values produced are the same field elements; the schedule is reorganised for the GPU:
//
//   a, b (and c = a o b) are written in natural order by the sparse mat-vec (qap.rs:37-58);
//   iNTT is a decimation-in-frequency transform  (natural in  -> bit-reversed out),
//   the coset scaling by g^i * n^-1 (qap.rs:63-70) is applied in bit-reversed position,
//   NTT  is a decimation-in-time transform       (bit-reversed in -> natural out),
// so no bit-reversal pass exists anywhere.  Stages are grouped into passes of <= 10 index bits; one CTA owns a
// 1024-element tile in shared memory (8 limb planes of u32, conflict-free for unit-stride butterflies) and runs all
// stages of its pass there.  The last inverse pass, the scaling and the first forward pass share a tile and are one
// kernel; the last forward pass also computes h = a*b - c (qap.rs:75-85) before storing.
#include "fp.cuh"
#include "ntt.cuh"
#include "util.cuh"

namespace b2g {

// 2^28-th root of unity 5^((r-1)/2^28) in Montgomery form (SURVEY.md App. A)
__device__ __forceinline__ fe fr_root_2_28() {
    fe r; r.l[0] = 0x80d13d9cu; r.l[1] = 0x636e7355u; r.l[2] = 0x2445ffd6u; r.l[3] = 0xa22bf374u;
    r.l[4] = 0x1eb203d8u; r.l[5] = 0x56452ac0u; r.l[6] = 0x2963f9e7u; r.l[7] = 0x1860ef94u;
    return r;
}

// pw[b] = omega_{2n}^(2^b), b = 0..logn ; ninv = n^-1
__global__ void ntt_setup_kernel(int logn, fe* __restrict__ pw, fe* __restrict__ ninv) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe g = fr_root_2_28();
    for (int i = 28; i > logn + 1; i--) g = Fr::sqr(g);
    for (int b = 0; b <= logn; b++) { pw[b] = g; g = Fr::sqr(g); }
    fe nn = fe_zero(); nn.l[0] = 1u << logn;          // logn <= 28
    *ninv = Fr::inv(Fr::from_canonical(nn));
}

// LibsnarkReduction coset: pg[b] = g^(2^b), pgi[b] = g^-(2^b) for g = 5 (Fr::GENERATOR), zinv = (g^n - 1)^-1
__global__ void ntt_setup_coset_kernel(int logn, fe* __restrict__ pg, fe* __restrict__ pgi, fe* __restrict__ zinv) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    fe five = fe_zero(); five.l[0] = 5;
    fe g = Fr::from_canonical(five), gi = Fr::inv(g);
    for (int b = 0; b <= logn; b++) { pg[b] = g; pgi[b] = gi; if (b < logn) { g = Fr::sqr(g); gi = Fr::sqr(gi); } }
    // after the loop g = 5^(2^logn) = g^n
    *zinv = Fr::inv(Fr::sub(g, Fr::one()));
}

// out[k] = scale * base^k for k < n, base^(2^b) given
__global__ void __launch_bounds__(256) ntt_powers_kernel(int logn, const fe* __restrict__ pw, const fe* __restrict__ scale, fe* __restrict__ out) {
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (1u << logn)) return;
    fe acc = *scale;
    for (int b = 0; b < logn; b++) if ((k >> b) & 1u) acc = Fr::mul(acc, pw[b]);
    fe_store(&out[k], acc);
}

// tw[k] = omega_{2n}^k, ct[k] = n^-1 * omega_{2n}^k, k < n
__global__ void __launch_bounds__(256) ntt_tables_kernel(int logn, const fe* __restrict__ pw, const fe* __restrict__ ninv,
                                                         fe* __restrict__ tw, fe* __restrict__ ct) {
    uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (1u << logn)) return;
    fe acc = Fr::one();
    for (int b = 0; b < logn; b++) if ((k >> b) & 1u) acc = Fr::mul(acc, pw[b]);
    fe_store(&tw[k], acc);
    fe_store(&ct[k], Fr::mul(acc, *ninv));
}

// ------------------------------------------------------------------------------------------------ sparse mat-vec
// a_i = <A_i, w>, b_i = <B_i, w> (evaluate_constraint, ark-groth16 0.5.0, called at qap.rs:42-43), c_i = a_i*b_i,
// a[m + j] = w[j] for j < num_inputs (qap.rs:46-50), everything else zero.  blockIdx.y = proof of a batch: its assignment
// starts at w + y * w_stride, its a, b, c at y * n.
__global__ void __launch_bounds__(256) spmv_kernel(uint32_t n, uint32_t m, uint32_t num_inputs, uint32_t w_stride,
                            const uint32_t* __restrict__ a_rowptr, const uint32_t* __restrict__ a_col, const fe* __restrict__ a_val,
                            const uint32_t* __restrict__ b_rowptr, const uint32_t* __restrict__ b_col, const fe* __restrict__ b_val,
                            const fe* __restrict__ w, fe* __restrict__ a, fe* __restrict__ b, fe* __restrict__ c,
                            const uint32_t* __restrict__ c_rowptr, const uint32_t* __restrict__ c_col, const fe* __restrict__ c_val) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    w += (size_t)blockIdx.y * w_stride;
    a += (size_t)blockIdx.y * n; b += (size_t)blockIdx.y * n; c += (size_t)blockIdx.y * n;
    fe ra = fe_zero(), rb = fe_zero(), rc = fe_zero();
    if (i < m) {
        const fe one = Fr::one();
        for (uint32_t k = a_rowptr[i]; k < a_rowptr[i + 1]; k++) {
            fe v = fe_load_nc(&a_val[k]); fe x = fe_load_nc(&w[a_col[k]]);
            ra = Fr::add(ra, fe_equal(v, one) ? x : Fr::mul(v, x));
        }
        for (uint32_t k = b_rowptr[i]; k < b_rowptr[i + 1]; k++) {
            fe v = fe_load_nc(&b_val[k]); fe x = fe_load_nc(&w[b_col[k]]);
            rb = Fr::add(rb, fe_equal(v, one) ? x : Fr::mul(v, x));
        }
        if (c_rowptr) {                                           // LibsnarkReduction: c from the real C matrix
            for (uint32_t k = c_rowptr[i]; k < c_rowptr[i + 1]; k++) {
                fe v = fe_load_nc(&c_val[k]); fe x = fe_load_nc(&w[c_col[k]]);
                rc = Fr::add(rc, fe_equal(v, one) ? x : Fr::mul(v, x));
            }
        } else {
            rc = Fr::mul(ra, rb);                                 // CircomReduction: c = a o b (qap.rs:52-58)
        }
    } else if (i < m + num_inputs) {
        ra = fe_load_nc(&w[i - m]);
    }
    fe_store(&a[i], ra); fe_store(&b[i], rb); fe_store(&c[i], rc);
}

// ------------------------------------------------------------------------------------------------ tiled passes
struct NttPassArgs {
    fe* vec[3];           // in-place vectors
    fe* out;              // pointwise result (h); may alias vec[0]
    const fe* tw;         // omega_{2n}^k, k < n
    const fe* ct;         // coset table applied by do_scale at the bit-reversed position: n^-1 * g^k
    const fe* pw_scale;   // optional scalar multiplied into the pointwise result (LibsnarkReduction: 1 / Z(g))
    int logn, tl;         // tl = log2(tile)
    int sb, k;            // transform bits [sb, sb + k) of the element index
    int do_dif, do_scale, do_dit, pointwise;
    size_t bstride;       // elements between the vectors of consecutive proofs of a batch (blockIdx.z = proof)
};

__device__ __forceinline__ uint32_t tile_global_index(uint32_t loc, uint32_t tile_id, int cols_log, int sb, int k) {
    uint32_t t = loc >> cols_log, col = loc & ((1u << cols_log) - 1u);
    uint32_t o = (tile_id << cols_log) | col;
    uint32_t lo = o & ((1u << sb) - 1u), high = o >> sb;
    return (high << (sb + k)) | (t << sb) | lo;
}

__device__ __forceinline__ fe sm_get(const uint32_t* sm, uint32_t tile, uint32_t i) {
    fe r;
    #pragma unroll
    for (int l = 0; l < 8; l++) r.l[l] = sm[l * tile + i];
    return r;
}
__device__ __forceinline__ void sm_put(uint32_t* sm, uint32_t tile, uint32_t i, const fe& v) {
    #pragma unroll
    for (int l = 0; l < 8; l++) sm[l * tile + i] = v.l[l];
}

// 2 CTAs/SM (<= 64 registers): with one 512-thread CTA per SM every stage barrier would idle the whole SM.  POINTWISE is a template parameter so that the plain passes do not carry the a*b accumulators.
template <bool POINTWISE>
__global__ void __launch_bounds__(512, 2) ntt_pass_kernel(NttPassArgs A) {
    extern __shared__ __align__(16) uint32_t sm[];
    const uint32_t tile = 1u << A.tl, half = tile >> 1, tid = threadIdx.x;
    const int cols_log = A.tl - A.k;
    const uint32_t n = 1u << A.logn;
    const uint32_t g0 = tile_global_index(tid, blockIdx.x, cols_log, A.sb, A.k);
    const uint32_t g1 = tile_global_index(tid + half, blockIdx.x, cols_log, A.sb, A.k);
    const int nv = POINTWISE ? 3 : 1;
    fe acc0 = fe_zero(), acc1 = fe_zero();
    const size_t zoff = (size_t)blockIdx.z * A.bstride;
    fe* const out = POINTWISE ? A.out + zoff : nullptr;
    for (int vi = 0; vi < nv; vi++) {
        fe* vec = (POINTWISE ? A.vec[vi] : A.vec[blockIdx.y]) + zoff;
        if (tid < half || half == 0) {
            sm_put(sm, tile, tid, fe_load(&vec[g0]));
            if (half) sm_put(sm, tile, tid + half, fe_load(&vec[g1]));
        }
        __syncthreads();
        if (A.do_dif) {
            for (int q = A.tl - 1; q >= cols_log; q--) {
                const int s = A.sb + (q - cols_log);                     // global stage: span 2^s
                if (tid < half) {
                    const uint32_t i0 = ((tid >> q) << (q + 1)) | (tid & ((1u << q) - 1u)), i1 = i0 + (1u << q);
                    const uint32_t gi = tile_global_index(i0, blockIdx.x, cols_log, A.sb, A.k);
                    const uint32_t j = gi & ((1u << s) - 1u);
                    const uint32_t e2 = j << (A.logn - s);               // 2 * (j * n / 2^(s+1))
                    fe u = sm_get(sm, tile, i0), v = sm_get(sm, tile, i1);
                    sm_put(sm, tile, i0, Fr::add(u, v));
                    fe d;
                    if (e2 == 0) d = Fr::sub(u, v);
                    else d = Fr::mul(Fr::sub(v, u), fe_load_nc(&A.tw[n - e2]));   // omega_n^-e = -omega_2n^(n-2e)
                    sm_put(sm, tile, i1, d);
                }
                __syncthreads();
            }
        }
        if (A.do_scale) {
            // position p holds coefficient bitrev(p): multiply by n^-1 * g^bitrev(p)   (qap.rs:63-70)
            if (tid < half || half == 0) {
                fe x = sm_get(sm, tile, tid);
                sm_put(sm, tile, tid, Fr::mul(x, fe_load_nc(&A.ct[A.logn ? __brev(g0) >> (32 - A.logn) : 0u])));
                if (half) {
                    fe y = sm_get(sm, tile, tid + half);
                    sm_put(sm, tile, tid + half, Fr::mul(y, fe_load_nc(&A.ct[A.logn ? __brev(g1) >> (32 - A.logn) : 0u])));
                }
            }
            __syncthreads();
        }
        if (A.do_dit) {
            for (int q = cols_log; q < A.tl; q++) {
                const int s = A.sb + (q - cols_log);
                if (tid < half) {
                    const uint32_t i0 = ((tid >> q) << (q + 1)) | (tid & ((1u << q) - 1u)), i1 = i0 + (1u << q);
                    const uint32_t gi = tile_global_index(i0, blockIdx.x, cols_log, A.sb, A.k);
                    const uint32_t j = gi & ((1u << s) - 1u);
                    const uint32_t e2 = j << (A.logn - s);
                    fe u = sm_get(sm, tile, i0), v = sm_get(sm, tile, i1);
                    if (e2 != 0) v = Fr::mul(v, fe_load_nc(&A.tw[e2]));
                    sm_put(sm, tile, i0, Fr::add(u, v));
                    sm_put(sm, tile, i1, Fr::sub(u, v));
                }
                __syncthreads();
            }
        }
        if (tid < half || half == 0) {
            fe x0 = sm_get(sm, tile, tid), x1 = half ? sm_get(sm, tile, tid + half) : fe_zero();
            if (!POINTWISE) {
                fe_store(&vec[g0], x0);
                if (half) fe_store(&vec[g1], x1);
            } else if (vi == 0) { acc0 = x0; acc1 = x1; }
            else if (vi == 1) { acc0 = Fr::mul(acc0, x0); acc1 = Fr::mul(acc1, x1); }
            else {
                fe r0 = Fr::sub(acc0, x0), r1 = Fr::sub(acc1, x1);        // h = a*b - c   (qap.rs:75-85)
                if (A.pw_scale) { const fe z = *A.pw_scale; r0 = Fr::mul(r0, z); r1 = Fr::mul(r1, z); }
                fe_store(&out[g0], r0);
                if (half) fe_store(&out[g1], r1);
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ radix-8 register passes
// [r2] Same butterflies, same twiddles, same results as ntt_pass_kernel above, reorganised so that the multiplier pipe is
// not waiting on shared memory and barriers: a thread keeps EIGHT elements in registers and runs up to three consecutive
// stages on them (a radix-8 "round") before the tile is exchanged through shared memory - 3-4 exchanges per pass instead
// of 10 barrier-separated stages, 1/3 of the shared-memory traffic, and the four twiddle loads of a step are in flight
// together.  Index bits: the thread's elements differ in a 3-bit field [f, f+3) of the tile-local index; a round on the
// stage bits [qa, qb) uses f = min(qa, tl-3).  Code size: every step pairs register POSITIONS (p, p+4); between steps the
// positions are rotated (x_new[p] = x_old[rotl3(p)], 64 register moves on the idle ALU pipe) so that ONE inlined copy of
// the four butterflies serves all three stage bits.  Position p holds field value rotl3^k(p).  Shared-memory index
// loc ^ (loc >> 3): conflict-free for every field position (tools/ntt8_model.py checks the schedule and the swizzle on CPU).
__device__ __forceinline__ uint32_t ntt8_sw(uint32_t loc) { return loc ^ (loc >> 3); }
__device__ __forceinline__ uint32_t ntt8_rotl3(uint32_t p) { return ((p << 1) | (p >> 2)) & 7u; }
__device__ __forceinline__ uint32_t ntt8_elem(uint32_t p, int k) {
    if (k >= 1) p = ntt8_rotl3(p);
    if (k == 2) p = ntt8_rotl3(p);
    return p;
}
__device__ __forceinline__ uint32_t ntt8_loc(uint32_t tid, uint32_t e, int f) {
    return ((tid >> f) << (f + 3)) | (e << f) | (tid & ((1u << f) - 1u));
}
// bring the position map to rotl3^want (k, want in {0,1,2})
__device__ __forceinline__ void ntt8_rotate_to(fe (&x)[8], int& k, int want) {
    const int d = (want - k + 3) % 3;
    if (d == 1) {            // x_new[p] = x_old[rotl3(p)] : 1<-2<-4<-1, 3<-6<-5<-3
        fe t = x[1]; x[1] = x[2]; x[2] = x[4]; x[4] = t;
        t = x[3]; x[3] = x[6]; x[6] = x[5]; x[5] = t;
    } else if (d == 2) {     // x_new[p] = x_old[rotr3(p)] : 1<-4<-2<-1, 3<-5<-6<-3
        fe t = x[1]; x[1] = x[4]; x[4] = x[2]; x[2] = t;
        t = x[3]; x[3] = x[5]; x[5] = x[6]; x[6] = t;
    }
    k = want;
}
__device__ __forceinline__ void ntt8_exchange(uint32_t* sm, uint32_t tile, uint32_t tid, fe (&x)[8], int f, int nf) {
    __syncthreads();                                           // everyone has read the previous exchange
    #pragma unroll
    for (int p = 0; p < 8; p++) sm_put(sm, tile, ntt8_sw(ntt8_loc(tid, p, f)), x[p]);
    __syncthreads();
    #pragma unroll
    for (int p = 0; p < 8; p++) x[p] = sm_get(sm, tile, ntt8_sw(ntt8_loc(tid, p, nf)));
}

template <bool POINTWISE>
__global__ void __launch_bounds__(256, 2) ntt_pass8_kernel(NttPassArgs A) {
    extern __shared__ __align__(16) uint32_t sm[];
    const uint32_t tile = 1u << A.tl, tid = threadIdx.x;
    const int cols_log = A.tl - A.k, ftop = A.tl - 3;
    const uint32_t n = 1u << A.logn;
    const int nv = POINTWISE ? 3 : 1;
    const size_t zoff = (size_t)blockIdx.z * A.bstride;
    fe* const out = POINTWISE ? A.out + zoff : nullptr;
    for (int vi = 0; vi < nv; vi++) {
        fe* vec = (POINTWISE ? A.vec[vi] : A.vec[blockIdx.y]) + zoff;
        fe x[8];
        int f = A.do_dif ? ftop : (cols_log < ftop ? cols_log : ftop), k = 0;
        #pragma unroll
        for (int p = 0; p < 8; p++) x[p] = fe_load(&vec[tile_global_index(ntt8_loc(tid, p, f), blockIdx.x, cols_log, A.sb, A.k)]);
        if (A.do_dif) {
            for (int qb = A.tl; qb > cols_log;) {
                const int qa = qb - 3 > cols_log ? qb - 3 : cols_log;
                const int nf = qa < ftop ? qa : ftop;
                if (nf != f) { ntt8_exchange(sm, tile, tid, x, f, nf); f = nf; }
                #pragma unroll 1
                for (int q = qb - 1; q >= qa; q--) {
                    ntt8_rotate_to(x, k, (q - f + 1) % 3);
                    const int s = A.sb + (q - cols_log);                 // global stage: span 2^s
                    #pragma unroll
                    for (int p = 0; p < 4; p++) {
                        const uint32_t gi = tile_global_index(ntt8_loc(tid, ntt8_elem(p, k), f), blockIdx.x, cols_log, A.sb, A.k);
                        const uint32_t e2 = (gi & ((1u << s) - 1u)) << (A.logn - s);
                        const fe u = x[p], v = x[p + 4];
                        x[p] = Fr::add(u, v);
                        if (e2 == 0) x[p + 4] = Fr::sub(u, v);
                        else x[p + 4] = Fr::mul(Fr::sub(v, u), fe_load_nc(&A.tw[n - e2]));   // omega_n^-e = -omega_2n^(n-2e)
                    }
                }
                ntt8_rotate_to(x, k, 0);
                qb = qa;
            }
        }
        if (A.do_scale) {
            // position g holds coefficient bitrev(g): multiply by n^-1 * g^bitrev(g)   (qap.rs:63-70)
            #pragma unroll 1
            for (int h = 0; h < 2; h++) {
                #pragma unroll
                for (int p = 0; p < 4; p++) {
                    const uint32_t g = tile_global_index(ntt8_loc(tid, p + 4 * h, f), blockIdx.x, cols_log, A.sb, A.k);
                    x[p] = Fr::mul(x[p], fe_load_nc(&A.ct[A.logn ? __brev(g) >> (32 - A.logn) : 0u]));
                }
                #pragma unroll
                for (int p = 0; p < 4; p++) { const fe t = x[p]; x[p] = x[p + 4]; x[p + 4] = t; }
            }
        }
        if (A.do_dit) {
            for (int qa = cols_log; qa < A.tl;) {
                const int qb = qa + 3 < A.tl ? qa + 3 : A.tl;
                const int nf = qa < ftop ? qa : ftop;
                if (nf != f) { ntt8_exchange(sm, tile, tid, x, f, nf); f = nf; }
                #pragma unroll 1
                for (int q = qa; q < qb; q++) {
                    ntt8_rotate_to(x, k, (q - f + 1) % 3);
                    const int s = A.sb + (q - cols_log);
                    #pragma unroll
                    for (int p = 0; p < 4; p++) {
                        const uint32_t gi = tile_global_index(ntt8_loc(tid, ntt8_elem(p, k), f), blockIdx.x, cols_log, A.sb, A.k);
                        const uint32_t e2 = (gi & ((1u << s) - 1u)) << (A.logn - s);
                        const fe u = x[p];
                        fe v = x[p + 4];
                        if (e2 != 0) v = Fr::mul(v, fe_load_nc(&A.tw[e2]));
                        x[p] = Fr::add(u, v);
                        x[p + 4] = Fr::sub(u, v);
                    }
                }
                ntt8_rotate_to(x, k, 0);
                qa = qb;
            }
        }
        // results: in place, or folded into h = a*b - c (qap.rs:75-85) with `out` as the running value (each thread re-reads
        // only what it wrote itself; out may alias vec[0])
        #pragma unroll 1
        for (int h = 0; h < 2; h++) {
            #pragma unroll
            for (int p = 0; p < 4; p++) {
                const uint32_t g = tile_global_index(ntt8_loc(tid, p + 4 * h, f), blockIdx.x, cols_log, A.sb, A.k);
                if (!POINTWISE) fe_store(&vec[g], x[p]);
                else if (vi == 0) fe_store(&out[g], x[p]);
                else if (vi == 1) fe_store(&out[g], Fr::mul(fe_load(&out[g]), x[p]));
                else {
                    fe r = Fr::sub(fe_load(&out[g]), x[p]);
                    if (A.pw_scale) r = Fr::mul(r, *A.pw_scale);
                    fe_store(&out[g], r);
                }
            }
            #pragma unroll
            for (int p = 0; p < 4; p++) { const fe t = x[p]; x[p] = x[p + 4]; x[p + 4] = t; }
        }
    }
}

// out[bitrev(i)] = in[i] * (scale ? *scale : 1); blockIdx.y = proof of a batch (vectors 2^logn apart)
__global__ void __launch_bounds__(256) bitrev_copy_kernel(const fe* __restrict__ in, fe* __restrict__ out, int logn, const fe* __restrict__ scale,
                                                          const fe* __restrict__ table) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (1u << logn)) return;
    in += (size_t)blockIdx.y << logn; out += (size_t)blockIdx.y << logn;
    uint32_t j = logn ? (__brev(i) >> (32 - logn)) : 0u;
    fe v = fe_load(&in[i]);
    if (scale) v = Fr::mul(v, *scale);
    if (table) v = Fr::mul(v, fe_load_nc(&table[j]));          // per-coefficient factor, indexed by the natural position
    fe_store(&out[j], v);
}

// ------------------------------------------------------------------------------------------------ host side
void ntt_domain_create(NttDomain& d, int logn, cudaStream_t st, bool libsnark) {
    // qap.rs:63-66 also needs the domain of size 2n, so n itself is limited to 2^27
    if (logn < 0 || logn > 27) throw_error(B2G_E_DOMAIN, "evaluation domain too large (PolynomialDegreeTooLarge)");
    d.logn = logn;
    const size_t n = (size_t)1 << logn;
    CUDA_CHECK(cudaMalloc(&d.tw, n * sizeof(fe)));
    CUDA_CHECK(cudaMalloc(&d.ct, n * sizeof(fe)));
    CUDA_CHECK(cudaMalloc(&d.pw, 32 * sizeof(fe)));
    ntt_setup_kernel<<<1, 1, 0, st>>>(logn, d.pw, d.pw + 30);
    ntt_tables_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logn, d.pw, d.pw + 30, d.tw, d.ct);
    if (libsnark) {
        CUDA_CHECK(cudaMalloc(&d.cg, n * sizeof(fe)));
        CUDA_CHECK(cudaMalloc(&d.cginv, n * sizeof(fe)));
        CUDA_CHECK(cudaMalloc(&d.zinv, 72 * sizeof(fe)));           // zinv | pg[32] | pgi[32]
        ntt_setup_coset_kernel<<<1, 1, 0, st>>>(logn, d.zinv + 1, d.zinv + 36, d.zinv);
        ntt_powers_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logn, d.zinv + 1, d.pw + 30, d.cg);
        ntt_powers_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logn, d.zinv + 36, d.pw + 30, d.cginv);
    }
    CUDA_CHECK(cudaGetLastError());
    // pass schedule: block pass (bits [0, tl)), then strided passes over the remaining bits, split evenly.
    // [r2] radix-8 register passes (ntt_pass8_kernel) from 2^5 up; B2G_NTT_RADIX2=1 keeps the one-stage-per-barrier kernel.
    // Tiles: 1024 elements (128 threads; B2G_NTT_TL = 5..11 overrides, 2048 elements = 256 threads).
    const char* r2 = getenv("B2G_NTT_RADIX2");
    d.radix8 = logn >= 5 && !(r2 && atoi(r2));
    int tlmax = 10;
    if (d.radix8) {
        if (const char* e = getenv("B2G_NTT_TL")) { int v = atoi(e); if (v >= 5 && v <= 11) tlmax = v; }
        CUDA_CHECK(cudaFuncSetAttribute(ntt_pass8_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        CUDA_CHECK(cudaFuncSetAttribute(ntt_pass8_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    }
    d.tl = logn < tlmax ? logn : tlmax;
    d.npass = 0;
    d.pass_sb[d.npass] = 0; d.pass_k[d.npass] = d.tl; d.pass_tl[d.npass] = d.tl; d.npass++;
    int rem = logn - d.tl;
    if (rem > 0) {
        // index bits per strided pass.  At 2^20 the three vectors (96 MB) already exceed the H100's 50 MB L2, but 2-D tiles
        // (B2G_NTT_MAXK=7) measured the same inside a whole 2^20 proof on an H100 (31.75 vs 31.84 proofs/s device-resident), so
        // the fewest passes (1024 x 1 tiles) stay up to 2^20.  From 2^21 on, strided tiles become 2-D with rows of >= 8
        // consecutive elements (256 B), i.e. <= 7 index bits per pass, so that no pass reads single 32-byte sectors at a
        // stride of 64 KB or more from DRAM.
        int maxk = logn > 20 && d.tl > 7 ? 7 : d.tl;
        if (const char* e = getenv("B2G_NTT_MAXK")) { int v = atoi(e); if (v >= 1 && v <= d.tl) maxk = v; }
        int np = (rem + maxk - 1) / maxk, sb = d.tl;
        if (np > 3) np = 3;                         // pass_sb / pass_k hold four entries
        for (int p = 0; p < np; p++) {
            int k = rem / (np - p);                 // even split
            int tl = d.tl;
            if (d.radix8) { tl = k > 10 ? k : 10; if (tl > logn) tl = logn; }
            d.pass_sb[d.npass] = sb; d.pass_k[d.npass] = k; d.pass_tl[d.npass] = tl; d.npass++;
            sb += k; rem -= k;
        }
    }
}

void ntt_domain_destroy(NttDomain& d) {
    if (d.tw) cudaFree(d.tw);
    if (d.ct) cudaFree(d.ct);
    if (d.pw) cudaFree(d.pw);
    if (d.cg) cudaFree(d.cg);
    if (d.cginv) cudaFree(d.cginv);
    if (d.zinv) cudaFree(d.zinv);
    d = NttDomain();
}

static void launch_pass(const NttDomain& d, fe* v0, fe* v1, fe* v2, int nvec, fe* out, int pass, int dif, int scale, int dit, int pointwise,
                        cudaStream_t st, const fe* coset_table = nullptr, const fe* pw_scale = nullptr, uint32_t count = 1) {
    NttPassArgs A;
    A.vec[0] = v0; A.vec[1] = v1; A.vec[2] = v2; A.out = out; A.tw = d.tw; A.ct = coset_table ? coset_table : d.ct; A.pw_scale = pw_scale;
    A.logn = d.logn; A.tl = d.pass_tl[pass]; A.sb = d.pass_sb[pass]; A.k = d.pass_k[pass];
    A.do_dif = dif; A.do_scale = scale; A.do_dit = dit; A.pointwise = pointwise; A.bstride = (size_t)1 << d.logn;
    const uint32_t tile = 1u << A.tl;
    const uint32_t ntiles = (uint32_t)(((size_t)1 << d.logn) >> A.tl);
    dim3 grid(ntiles, pointwise ? 1 : nvec, count);
    if (d.radix8) {
        if (pointwise) ntt_pass8_kernel<true><<<grid, tile / 8, tile * 32, st>>>(A);
        else ntt_pass8_kernel<false><<<grid, tile / 8, tile * 32, st>>>(A);
    } else {
        uint32_t threads = tile / 2 ? tile / 2 : 1;
        if (pointwise) ntt_pass_kernel<true><<<grid, threads, tile * 32, st>>>(A);
        else ntt_pass_kernel<false><<<grid, threads, tile * 32, st>>>(A);
    }
    g_launch_count += 1;
}

// the three vectors a, b, c (natural order, in place) -> h (natural order) in `out`; `count` proofs whose vectors are n apart
void ntt_witness_transform(const NttDomain& d, fe* a, fe* b, fe* c, fe* out, cudaStream_t st, uint32_t count) {
    for (int p = d.npass - 1; p >= 1; p--) launch_pass(d, a, b, c, 3, nullptr, p, 1, 0, 0, 0, st, nullptr, nullptr, count);
    const bool single = d.npass == 1;
    launch_pass(d, a, b, c, 3, out, 0, 1, 1, 1, single ? 1 : 0, st, nullptr, nullptr, count);
    for (int p = 1; p < d.npass; p++) launch_pass(d, a, b, c, 3, out, p, 0, 0, 1, p == d.npass - 1 ? 1 : 0, st, nullptr, nullptr, count);
    CUDA_CHECK(cudaGetLastError());
}

// ONE vector through the same chain, in place and without the pointwise step: evaluations on H (natural order) ->
// coefficients -> evaluations on the coset g*H (natural order).  Used when the three transforms of a proof run on three
// different GPUs (prover.cu, sharded proofs) and h = a*b - c is formed from peer memory afterwards.
void ntt_transform_single(const NttDomain& d, fe* v, cudaStream_t st) {
    for (int p = d.npass - 1; p >= 1; p--) launch_pass(d, v, nullptr, nullptr, 1, nullptr, p, 1, 0, 0, 0, st);
    launch_pass(d, v, nullptr, nullptr, 1, nullptr, 0, 1, 1, 1, 0, st);
    for (int p = 1; p < d.npass; p++) launch_pass(d, v, nullptr, nullptr, 1, nullptr, p, 0, 0, 1, 0, st);
    CUDA_CHECK(cudaGetLastError());
}

// LibsnarkReduction::witness_map_from_matrices (ark-groth16 0.5.0 r1cs_to_qap.rs, the default QAP of Groth16<Bn254> used by
// /root/reference/tests/groth16.rs): a, b, c (c from the real C matrix) -> coefficients -> evaluations on the coset
// g*H (g = 5) -> (a*b - c) / Z(g) -> coset iFFT -> the n coefficients of h, natural order, in `out`.
// Same kernels as the Circom map; the coset tables are cg / cginv, and the last inverse transform is a DIF pass set
// followed by one bit-reversing copy that applies n^-1 g^-i.
void ntt_witness_transform_libsnark(const NttDomain& d, fe* a, fe* b, fe* c, fe* scratch, fe* out, cudaStream_t st, uint32_t count) {
    if (!d.cg) throw_error(B2G_E_SHAPE, "matrices were not loaded for LibsnarkReduction");
    for (int p = d.npass - 1; p >= 1; p--) launch_pass(d, a, b, c, 3, nullptr, p, 1, 0, 0, 0, st, nullptr, nullptr, count);
    const bool single = d.npass == 1;
    launch_pass(d, a, b, c, 3, scratch, 0, 1, 1, 1, single ? 1 : 0, st, d.cg, d.zinv, count);
    for (int p = 1; p < d.npass; p++) launch_pass(d, a, b, c, 3, scratch, p, 0, 0, 1, p == d.npass - 1 ? 1 : 0, st, d.cg, d.zinv, count);
    for (int p = d.npass - 1; p >= 0; p--) launch_pass(d, scratch, nullptr, nullptr, 1, nullptr, p, 1, 0, 0, 0, st, nullptr, nullptr, count);
    const size_t n = (size_t)1 << d.logn;
    bitrev_copy_kernel<<<dim3((unsigned)((n + 255) / 256), count), 256, 0, st>>>(scratch, out, d.logn, nullptr, d.cginv);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

// plain natural-order (i)NTT of one vector (parity entry point b2g_ntt); tmp = scratch of n elements
void ntt_plain(const NttDomain& d, fe* data, fe* tmp, bool inverse, cudaStream_t st) {
    const size_t n = (size_t)1 << d.logn;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    if (inverse) {
        for (int p = d.npass - 1; p >= 0; p--) launch_pass(d, data, nullptr, nullptr, 1, nullptr, p, 1, 0, 0, 0, st);
        bitrev_copy_kernel<<<blocks, 256, 0, st>>>(data, tmp, d.logn, d.ct, nullptr);   // ct[0] = n^-1
        CUDA_CHECK(cudaMemcpyAsync(data, tmp, n * sizeof(fe), cudaMemcpyDeviceToDevice, st));
    } else {
        bitrev_copy_kernel<<<blocks, 256, 0, st>>>(data, tmp, d.logn, nullptr, nullptr);
        CUDA_CHECK(cudaMemcpyAsync(data, tmp, n * sizeof(fe), cudaMemcpyDeviceToDevice, st));
        for (int p = 0; p < d.npass; p++) launch_pass(d, data, nullptr, nullptr, 1, nullptr, p, 0, 0, 1, 0, st);
    }
    CUDA_CHECK(cudaGetLastError());
}

void ntt_powers(int logn, const fe* pw, const fe* scale, fe* out, cudaStream_t st) {
    const size_t n = (size_t)1 << logn;
    ntt_powers_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logn, pw, scale, out);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

void spmv_launch(uint32_t n, uint32_t m, uint32_t num_inputs, const uint32_t* a_rowptr, const uint32_t* a_col, const fe* a_val,
                 const uint32_t* b_rowptr, const uint32_t* b_col, const fe* b_val, const fe* w, fe* a, fe* b, fe* c, cudaStream_t st,
                 const uint32_t* c_rowptr, const uint32_t* c_col, const fe* c_val, uint32_t count, uint32_t w_stride) {
    spmv_kernel<<<dim3((n + 255) / 256, count), 256, 0, st>>>(n, m, num_inputs, w_stride, a_rowptr, a_col, a_val, b_rowptr, b_col, b_val, w, a, b, c, c_rowptr, c_col, c_val);
    g_launch_count += 1;
    CUDA_CHECK(cudaGetLastError());
}

}  // namespace b2g
