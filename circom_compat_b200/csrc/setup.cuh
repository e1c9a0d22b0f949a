// setup.cuh - what the context code (prover.cu), the device setup (setup.cu) and the key check (ptau.cu) share about a circuit.
#pragma once
#include <algorithm>
#include <string>
#include <cuda_runtime.h>
#include "../../include/b2groth.h"
#include "fp.cuh"
#include "util.cuh"

namespace b2g {

// The checks of a matrix descriptor that b2g_matrices_load and b2g_setup share (each caller checks its own pointers first).
// with_c: the C matrix is required and read whatever the reduction (b2g_setup); otherwise only LibsnarkReduction reads it.
// Returns log2 of the domain, the least power of two >= num_constraints + num_inputs.  Defined in prover.cu.
int mat_desc_check(const b2g_mat_desc* d, bool with_c);

// mat_desc_check with C for a setup or key check, whose CircomReduction H query transforms over 2n points
inline int setup_domain(const b2g_mat_desc* d) {
    const int logn = mat_desc_check(d, true);
    if (d->reduction != B2G_REDUCTION_LIBSNARK && logn > 26)
        throw_error(B2G_E_DOMAIN, "PolynomialDegreeTooLarge: a CircomReduction setup transforms over 2n points, so n must fit 2^26");
    return logn;
}

// the nonzeros of matrix x (0 A, 1 B, 2 C)
inline uint32_t mat_nnz(const b2g_mat_desc* d, int x) {
    return (x == 0 ? d->a_rowptr : x == 1 ? d->b_rowptr : d->c_rowptr)[d->num_constraints];
}

// the most nonzeros of one matrix, which cub's int counts bound; fn names the entry point in the message
inline uint32_t max_nnz(const b2g_mat_desc* d, const char* fn) {
    const uint32_t most = std::max(mat_nnz(d, 0), std::max(mat_nnz(d, 1), mat_nnz(d, 2)));
    if (most > (uint32_t)INT32_MAX) throw_error(B2G_E_DEVICE, std::string(fn) + ": more than 2^31 - 1 nonzeros in one matrix");
    return most;
}

// copies matrix x into the caller's device buffers: rowptr (num_constraints + 1 words), col and val (mat_nnz each)
inline void mat_upload(const b2g_mat_desc* d, int x, uint32_t* rowptr, uint32_t* col, fe* val, cudaStream_t st) {
    const uint32_t* rp = x == 0 ? d->a_rowptr : x == 1 ? d->b_rowptr : d->c_rowptr;
    const uint32_t* cl = x == 0 ? d->a_col : x == 1 ? d->b_col : d->c_col;
    const void* vl = x == 0 ? d->a_val : x == 1 ? d->b_val : d->c_val;
    const uint32_t m = d->num_constraints, nnz = rp[m];
    CUDA_CHECK(cudaMemcpyAsync(rowptr, rp, ((size_t)m + 1) * 4, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(col, cl, (size_t)nnz * 4, cudaMemcpyHostToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(val, vl, (size_t)nnz * sizeof(fe), cudaMemcpyHostToDevice, st));
}

// the row of nonzero p: the last row r < m with rowptr[r] <= p (rowptr[m] = nnz > p), in log2(m) steps however long the row
__device__ __forceinline__ uint32_t mat_row(const uint32_t* __restrict__ rowptr, uint32_t m, uint32_t p) {
    uint32_t lo = 0, hi = m - 1;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (rowptr[mid] <= p) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// out[key] = the Fr sum of the n products prod[k] with keys[k] = key, for the keys that occur (keys sorted): a reduce-by-key
// into uniq and agg, the run count at *runs (device), then a scatter.  With temp null, only sets temp_bytes.  (setup.cu)
void sum_by_key(void* temp, size_t& temp_bytes, const uint32_t* keys, uint32_t* uniq, const fe* prod, fe* agg, uint32_t* runs,
                uint32_t n, fe* out, cudaStream_t st);

// b2g_test_op op SCALE_SPLIT_TEST_OP: b2g_points_scale's G1 and G2 scalar splits (contribute.cu)
constexpr int SCALE_SPLIT_TEST_OP = 54;
void scale_split_test_op(cudaStream_t st, const void* a, size_t n, void* out);

}  // namespace b2g
