// verify.cuh - what the context code (prover.cu) and the batched verifier (verify.cu) share.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

struct b2g_ctx;

namespace b2g {

struct VerifyBufs;                          // a context's b2g_verify_many buffers (verify.cu)
void verify_bufs_free(VerifyBufs* v);

// the parts of a context verify.cu uses (b2g_ctx is private to prover.cu)
struct CtxView { int device; cudaStream_t st; bool proof_pending; VerifyBufs** vbufs; };
CtxView ctx_view(b2g_ctx* ctx);
// ctx_view of a context with no submitted proof pending; B2G_E_SHAPE otherwise
CtxView ctx_idle(b2g_ctx* ctx);

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

// b2g_powers_check's point rules over the n affine Montgomery points of a device slice whose first point has index `base` in its
// array: atomicMin of the index of every point with a coordinate >= p, off its curve, at infinity, outside G2 (G2 only) or, with
// `gen`, other than the generator at index 0, into *bad (device).  Asynchronous.
void powers_rules(bool g2, const void* pts, uint32_t n, uint64_t base, bool gen, unsigned long long* bad, cudaStream_t st);
// the first of those rules the one device point at pt breaks: 1 a coordinate >= p, 2 off its curve, 3 at infinity, 4 outside
// G2, 5 not the generator (only with gen); 0 when it passes.  scratch: 4 device bytes.  Synchronises the stream.
uint32_t powers_point_rule(bool g2, const void* pt, bool gen, uint32_t* scratch, cudaStream_t st);
// b2g_powers_check's pairing product (include/b2groth.h) into *verdict (device, 1 or 0).  sums = S_T, S_A, S_B (G1 XYZZ, 128 B
// each), S_U (G2 XYZZ); g1 = T_0, T_1, T_(2n-2), A_0, A_(n-1), B_0, B_(n-1); g2 = U_0, U_1, U_(n-1), beta_2 (affine Montgomery);
// ch = rho, sigma, pi, kappa, eps (32 B canonical each); all device.  Asynchronous.
void powers_verdict(const void* sums, const void* g1, const void* g2, const void* ch, uint32_t log_n, uint32_t* verdict, cudaStream_t st);

// b2g_setup_check's point rules over the n affine Montgomery points of a device slice whose first point has index `base` in its
// array: atomicMin of the index of every point with a coordinate >= p, off its curve or, for G2, outside G2, into *bad (device).
// Infinity passes.  Asynchronous.
void setup_rules(bool g2, const void* pts, uint32_t n, uint64_t base, unsigned long long* bad, cudaStream_t st);
// b2g_setup_check's sums, XYZZ records at these byte offsets of one device buffer of SC_BYTES (G1 128 B, G2 256 B): the key
// side sum_j rho^j X_j of a_query, b_g1_query, b_g2_query, gamma_abc_g1, l_query (from rho^ni) and sum_i sigma^i h_query[i];
// the ceremony side sum_k s_k Y_k of E1 (s^A T), E2 (s^B T), E3 (s^B U), E4 (s^A Be, s^B Al, s^C T) and E5 (h T)
enum : size_t {
    SC_KA = 0, SC_KB1 = 128, SC_KB2 = 256, SC_KIC = 512, SC_KL = 640, SC_KH = 768,
    SC_RA = 896, SC_RB1 = 1024, SC_RB2 = 1152, SC_RBE = 1408, SC_RAL = 1536, SC_RC = 1664, SC_RH = 1792, SC_BYTES = 1920
};
// b2g_setup_check's equations E1-E6 (include/b2groth.h) into *verdict (device): the lowest failing equation 1-6, or 0.
// sums: the SC_ records; g1 = delta_1, T_0; g2 = gamma_2, delta_2, U_0 (affine Montgomery); all device.  Asynchronous.
void setup_check_verdict(const void* sums, const void* g1, const void* g2, uint32_t* verdict, cudaStream_t st);

}  // namespace b2g
