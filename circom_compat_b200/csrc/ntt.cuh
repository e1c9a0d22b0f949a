// ntt.cuh - host-visible interface of ntt.cu (radix-2 domain tables, witness-map transforms, sparse mat-vec).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "fp.cuh"

namespace b2g {

struct NttDomain {
    int logn = -1, tl = 0, npass = 0;
    int pass_sb[4] = {0, 0, 0, 0}, pass_k[4] = {0, 0, 0, 0}, pass_tl[4] = {0, 0, 0, 0};
    bool radix8 = false;                                      // ntt_pass8_kernel (register radix-8 rounds) instead of ntt_pass_kernel
    fe *tw = nullptr, *ct = nullptr, *pw = nullptr;
    // LibsnarkReduction only: coset by the field generator g = 5 (ark-poly get_coset(F::GENERATOR))
    fe *cg = nullptr, *cginv = nullptr, *zinv = nullptr;      // n^-1 g^k, n^-1 g^-k (k < n), (g^n - 1)^-1
};

void ntt_domain_create(NttDomain& d, int logn, cudaStream_t st, bool libsnark = false);
void ntt_domain_destroy(NttDomain& d);
// an NttDomain of 2^logn points that is destroyed with its holder, also when its creation fails part way
struct NttDomainHold : NttDomain {
    NttDomainHold(int logn, cudaStream_t st) {
        try { ntt_domain_create(*this, logn, st); } catch (...) { ntt_domain_destroy(*this); throw; }
    }
    NttDomainHold(const NttDomainHold&) = delete;
    NttDomainHold& operator=(const NttDomainHold&) = delete;
    ~NttDomainHold() { ntt_domain_destroy(*this); }
};
// count > 1: a batch of proofs whose vectors lie 2^logn elements apart (b2g_prove_many)
void ntt_witness_transform(const NttDomain& d, fe* a, fe* b, fe* c, fe* out, cudaStream_t st, uint32_t count = 1);
void ntt_transform_single(const NttDomain& d, fe* v, cudaStream_t st);
void ntt_witness_transform_libsnark(const NttDomain& d, fe* a, fe* b, fe* c, fe* scratch, fe* out, cudaStream_t st, uint32_t count = 1);
void ntt_plain(const NttDomain& d, fe* data, fe* tmp, bool inverse, cudaStream_t st);
// out[k] = *scale * x^k for k < 2^logn, from pw[b] = x^(2^b), b < logn (device pointers)
void ntt_powers(int logn, const fe* pw, const fe* scale, fe* out, cudaStream_t st);
void spmv_launch(uint32_t n, uint32_t m, uint32_t num_inputs, const uint32_t* a_rowptr, const uint32_t* a_col, const fe* a_val,
                 const uint32_t* b_rowptr, const uint32_t* b_col, const fe* b_val, const fe* w, fe* a, fe* b, fe* c, cudaStream_t st,
                 const uint32_t* c_rowptr = nullptr, const uint32_t* c_col = nullptr, const fe* c_val = nullptr,
                 uint32_t count = 1, uint32_t w_stride = 0);       // count assignments w_stride apart -> a, b, c of count x n

}  // namespace b2g
