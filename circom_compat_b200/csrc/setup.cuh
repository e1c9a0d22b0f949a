// setup.cuh - what the context code (prover.cu) and the device setup (setup.cu) share.
#pragma once
#include <cuda_runtime.h>
#include "../../include/b2groth.h"

namespace b2g {

// The checks of a matrix descriptor that b2g_matrices_load and b2g_setup share (each caller checks its own pointers first).
// with_c: the C matrix is required and read whatever the reduction (b2g_setup); otherwise only LibsnarkReduction reads it.
// Returns log2 of the domain, the least power of two >= num_constraints + num_inputs.  Defined in prover.cu.
int mat_desc_check(const b2g_mat_desc* d, bool with_c);

// b2g_test_op op SCALE_SPLIT_TEST_OP: b2g_points_scale's G1 and G2 scalar splits (contribute.cu)
constexpr int SCALE_SPLIT_TEST_OP = 54;
void scale_split_test_op(cudaStream_t st, const void* a, size_t n, void* out);

}  // namespace b2g
