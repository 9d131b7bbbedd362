// NF4 weights of the decoder's projections (bitsandbytes' blockwise 4-bit format, blocksize 64, fp32 absmax, no
// double quantisation; oracle/nf4_ref.py restates it).  A weight [N, K] holds codes [N, K / 2] (two per byte, the
// first element in the high nibble) and absmax [N, K / 64]; element (n, k) is fp16(kNF4[q] * absmax[n][k / 64]).
#pragma once
#include <cuda_fp16.h>
#include "rmu_common.h"
#include "rmu_gemm.cuh"

namespace rmu {

constexpr int kNf4Block = 64;

struct Nf4Weight {
    uint8_t* codes = nullptr;             // [rows, cols / 2]
    float* absmax = nullptr;              // [rows, cols / 64]
    int rows = 0, cols = 0;
};

// the quantiser: fp16 hi [n] (n a multiple of 64) -> packed codes [n / 2] and absmax [n / 64], bit-identical to
// nf4_ref.quantize
int launch_nf4_quantize(const __half* hi, int64_t n, uint8_t* codes, float* absmax, cudaStream_t st);
// hi [n] = fp16(code * absmax) (nf4_ref.dequantize); the matching lo plane is the caller's zeros
int launch_nf4_dequantize(const uint8_t* codes, const float* absmax, int64_t n, __half* hi, cudaStream_t st);
// the decode GEMV: out[n] for one row x = x_hi + x_lo [K] against W [N, K] in NF4, with E1's epilogue `mode`
// (GEMM_BIAS_F32, GEMM_BIAS_RESF32_F32 or GEMM_BIAS_SWIGLU_SPLIT; p.M must be 1).  N % 128 == 0, K % 64 == 0 and
// K <= kNf4MaxK; the caller checks them.
constexpr int kNf4MaxK = 49152;           // x staged in shared memory as fp32: 192 KB
int launch_nf4_gemv(int mode, const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p,
                    int sms, cudaStream_t st);
// the same GEMV on p.M <= kNf4MaxRows rows x [M, K] (row pitch K; out row pitch p.out_ld, or N, N / 2 for SwiGLU),
// each row's bits those of launch_nf4_gemv on that row alone
constexpr int kNf4MaxRows = 16;
int launch_nf4_gemv_rows(int mode, const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p,
                         int sms, cudaStream_t st);

}  // namespace rmu
