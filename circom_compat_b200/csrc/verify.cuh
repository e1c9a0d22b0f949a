// verify.cuh - what the context code (prover.cu) and the batched verifier (verify.cu) share.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

struct b2g_ctx;

namespace b2g {

struct VerifyBufs;                          // a context's b2g_verify_many buffers (verify.cu)
void verify_bufs_free(VerifyBufs* v);

// the parts of a context verify.cu uses (b2g_ctx is private to prover.cu)
struct CtxView { int device; cudaStream_t st; bool proof_pending; VerifyBufs** vbufs; };
CtxView ctx_view(b2g_ctx* ctx);

// b2g_test_op ops PAIRING_TEST_OP0 and up: the Fq12 tower and the pairing (verify.cu)
constexpr int PAIRING_TEST_OP0 = 30;
void pairing_test_op(cudaStream_t st, int op, const void* a, const void* b, size_t n, void* out);

// b2g_setup's generator checks on a device buffer of a G1 (64 B) and a G2 (128 B) affine Montgomery point; a NULL pointer is
// not checked.  Returns 0, or 1 for a G1 point at infinity or off its curve, 2 for a G2 point at infinity or off its twist, 3 for
// a G2 point outside G2.  Synchronises the stream.
int setup_generators_check(const void* g1, const void* g2, cudaStream_t st);

// The lowest i < n whose point in the device buffer pts (n affine Montgomery G1 or G2 points, zeros = infinity) has a coordinate
// >= p or lies off its curve (*why = 1), or, with `subgroup`, is a G2 point outside G2 (*why = 2); n when every point passes.
// Synchronises the stream.
uint64_t points_check(bool g2, const void* pts, size_t n, bool subgroup, cudaStream_t st, int* why);

}  // namespace b2g
