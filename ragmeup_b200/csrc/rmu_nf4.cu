// NF4 decoder weights (rmu_nf4.cuh): the quantiser, the dequantiser of the prefill and the decode GEMV.
#include <algorithm>

#include "rmu_nf4.cuh"

namespace rmu {

// Dettmers et al., QLoRA (2023), Appendix E; bitsandbytes' NF4 table in fp32 (oracle/nf4_ref.py CODE)
__device__ const float kNF4[16] = {
    -1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,
    -0.18477343022823334f, -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f,
    0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f,
    0.7229568362236023f, 1.0f};

// bitsandbytes' dQuantizeNF4: its threshold tree with strict '>' answers the number of thresholds below x (NaN, the
// scaled value of an all-zero block, passes none: code 0)
__device__ __forceinline__ unsigned nf4_code(float x) {
    const float t[15] = {-0.8480964004993439f, -0.6106329262256622f, -0.4599952697753906f, -0.33967943489551544f,
                         -0.23460740596055984f, -0.13791173323988914f, -0.045525018125772476f, 0.03979014977812767f,
                         0.1202552504837513f, 0.2035212516784668f, 0.2920137718319893f, 0.3893125355243683f,
                         0.5016634166240692f, 0.6427869200706482f, 0.8614784181118011f};
    unsigned q = 0;
#pragma unroll
    for (int i = 0; i < 15; ++i) q += x > t[i] ? 1u : 0u;
    return q;
}

// one warp per 64-element block: lane l holds elements 2l, 2l + 1 and writes their byte
__global__ void __launch_bounds__(256) nf4_quantize_kernel(const __half* __restrict__ hi, int64_t nblocks,
                                                           uint8_t* __restrict__ codes, float* __restrict__ absmax) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
    if (b >= nblocks) return;
    const unsigned lane = threadIdx.x & 31;
    const float2 f = __half22float2(reinterpret_cast<const __half2*>(hi + b * kNf4Block)[lane]);
    float m = fmaxf(fabsf(f.x), fabsf(f.y));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float inv = __frcp_rn(m);                                   // 1 / absmax, inf for an all-zero block
    codes[b * 32 + lane] = static_cast<uint8_t>((nf4_code(__fmul_rn(f.x, inv)) << 4) | nf4_code(__fmul_rn(f.y, inv)));
    if (lane == 0) absmax[b] = m;
}

// one thread per 8 elements (4 code bytes -> 8 halves)
__global__ void __launch_bounds__(256) nf4_dequantize_kernel(const uint32_t* __restrict__ codes,
                                                             const float* __restrict__ absmax, int64_t n8,
                                                             uint4* __restrict__ hi) {
    __shared__ float tab[16];
    if (threadIdx.x < 16) tab[threadIdx.x] = kNF4[threadIdx.x];
    __syncthreads();
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const uint32_t c = codes[i];
        const float a = __ldg(absmax + (i >> 3));
        uint4 out;
        uint32_t* o = reinterpret_cast<uint32_t*>(&out);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const unsigned byte = (c >> (8 * j)) & 255u;
            const __half2 h = __floats2half2_rn(__fmul_rn(tab[byte >> 4], a), __fmul_rn(tab[byte & 15u], a));
            o[j] = *reinterpret_cast<const uint32_t*>(&h);
        }
        hi[i] = out;
    }
}

// The decode GEMV.  One warp per row pair (r0, r0 + 64) with r0 = 128 (p / 64) + p % 64: SwiGLU's gate row and its
// up row (E1's 64 + 64 row blocks), so output column p is one warp's; the other modes use the same pairing.  Lane l
// reads 16-byte chunks l, l + 32, .. of both rows' codes (32 weights each, half a quantisation block, one absmax) and
// accumulates w * x in fp32 in chunk order, then a butterfly sums the lanes: the order is fixed, so a repeat gives
// the same bits.  Each weight is fp16(code * absmax), the value the dequantiser writes for the prefill; x = hi + lo
// is staged once per CTA in shared memory as fp32.
//
// Lane l reads its chunk's 32 x values as eight 16-byte units, and the chunks of neighbouring lanes lie 128 bytes
// apart: stored in order, the eight lanes of a quarter-warp would all hit one 16-byte bank group (8-way conflicts).
// Unit j of chunk c is therefore stored at unit 8 c + (j ^ (c & 7)), which spreads them over all eight groups.
constexpr int kGemvThreads = 256, kGemvPairs = kGemvThreads / 32, kGemvCtasPerSm = 4;

// the float index where x[k] is staged
__device__ __forceinline__ int nf4_x_slot(int k) { return (((k >> 2) ^ ((k >> 5) & 7)) << 2) | (k & 3); }

// xv: chunk c's eight units, sw = c & 7
__device__ __forceinline__ void nf4_dot16(const uint4& u, float s, const float4* xv, int sw, const float* tab,
                                          float& acc) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 xa = xv[(2 * j) ^ sw], xb = xv[(2 * j + 1) ^ sw];
        const float xx[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const unsigned byte = (w[j] >> (8 * b)) & 255u;
            const float2 f = __half22float2(__floats2half2_rn(__fmul_rn(tab[byte >> 4], s), __fmul_rn(tab[byte & 15u], s)));
            acc = fmaf(f.x, xx[2 * b], acc);
            acc = fmaf(f.y, xx[2 * b + 1], acc);
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(kGemvThreads, kGemvCtasPerSm)
nf4_gemv_kernel(const __half* __restrict__ x_hi, const __half* __restrict__ x_lo, const uint8_t* __restrict__ codes,
                const float* __restrict__ absmax, const GemmParams p) {
    extern __shared__ float4 nf4_x4[];
    float* xs = reinterpret_cast<float*>(nf4_x4);                      // [K]
    __shared__ float tab[16];
    const int K = p.K;
    if (threadIdx.x < 16) tab[threadIdx.x] = kNF4[threadIdx.x];
    for (int k = 2 * threadIdx.x; k < K; k += 2 * kGemvThreads) {
        const float2 h = __half22float2(*reinterpret_cast<const __half2*>(x_hi + k));
        const float2 l = __half22float2(*reinterpret_cast<const __half2*>(x_lo + k));
        *reinterpret_cast<float2*>(xs + nf4_x_slot(k)) = make_float2(h.x + l.x, h.y + l.y);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = K / 32, pairs = p.N / 2;
    const size_t row_chunks = static_cast<size_t>(chunks), row_blocks = static_cast<size_t>(K / kNf4Block);
    const uint4* c4 = reinterpret_cast<const uint4*>(codes);
    for (int pi = blockIdx.x * kGemvPairs + warp; pi < pairs; pi += gridDim.x * kGemvPairs) {
        const int r0 = 128 * (pi >> 6) + (pi & 63), r1 = r0 + 64;
        const uint4* c0 = c4 + r0 * row_chunks;
        const uint4* c1 = c4 + r1 * row_chunks;
        const float* a0 = absmax + r0 * row_blocks;
        const float* a1 = absmax + r1 * row_blocks;
        float acc0 = 0.f, acc1 = 0.f;
        int ch = lane;
        uint4 u0{}, u1{};
        float s0 = 0.f, s1 = 0.f;
        if (ch < chunks) { u0 = __ldcs(c0 + ch); u1 = __ldcs(c1 + ch); s0 = __ldg(a0 + (ch >> 1)); s1 = __ldg(a1 + (ch >> 1)); }
        while (ch < chunks) {
            const int nx = ch + 32;
            uint4 v0{}, v1{};
            float t0 = 0.f, t1 = 0.f;
            if (nx < chunks) { v0 = __ldcs(c0 + nx); v1 = __ldcs(c1 + nx); t0 = __ldg(a0 + (nx >> 1)); t1 = __ldg(a1 + (nx >> 1)); }
            const float4* xv = reinterpret_cast<const float4*>(xs + 32 * ch);
            nf4_dot16(u0, s0, xv, ch & 7, tab, acc0);
            nf4_dot16(u1, s1, xv, ch & 7, tab, acc1);
            u0 = v0; u1 = v1; s0 = t0; s1 = t1;
            ch = nx;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
            acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
        }
        if (lane != 0) continue;
        // E1's epilogues at M = 1, in its order of operations
        if constexpr (MODE == GEMM_BIAS_SWIGLU_SPLIT) {
            const float g = acc0 + p.bias[r0];
            const float v = g / (1.0f + expf(-g)) * (acc1 + p.bias[r1]);
            __half h, l;
            split_f16(v, h, l);
            p.out_hi[pi] = h;
            p.out_lo[pi] = l;
            if (p.range_flag && !(fabsf(v) <= 65504.0f)) atomicOr(p.range_flag, 1);
        } else {
            float v0 = acc0 + p.bias[r0], v1 = acc1 + p.bias[r1];
            if constexpr (MODE == GEMM_BIAS_RESF32_F32) {
                v0 = v0 + p.res_f32[r0];
                v1 = v1 + p.res_f32[r1];
            }
            p.out_f32[r0] = v0;
            p.out_f32[r1] = v1;
        }
    }
}

// The batched decode's GEMV: rows m < M (M <= MM <= kNf4MaxRows) of x [M, K] (row pitch K) against W, one read of
// the codes and absmax for every row.  Same warp-per-row-pair layout and chunk order as nf4_gemv_kernel: lane l still
// takes chunks l, l + 32, .., each dequantised once into registers with nf4_dot16's operations, then each row's fp32
// chain over the chunk's 32 weights in element order, then the same butterfly, so row m's bits are those of an M = 1
// launch on row m.  x is staged in K-slices of 1024 values (32 chunks, one per lane, nf4_x_slot's swizzle within the
// slice) for all M rows at once: M x 4 KB of shared memory at any K.
constexpr int kNf4SliceK = 1024;

// CTAs per SM the row GEMV is compiled for: 16 rows of accumulators need more than 128 registers a thread
constexpr int gemv_rows_ctas(int mm) { return mm > 8 ? 1 : 2; }

template <int MODE, int MM>
__global__ void __launch_bounds__(kGemvThreads, gemv_rows_ctas(MM))
nf4_gemv_rows_kernel(const __half* __restrict__ x_hi, const __half* __restrict__ x_lo, int M,
                     const uint8_t* __restrict__ codes, const float* __restrict__ absmax, const GemmParams p) {
    extern __shared__ float4 nf4_xr4[];
    float* xs = reinterpret_cast<float*>(nf4_xr4);                     // [M][kNf4SliceK]
    __shared__ float tab[16];
    const int K = p.K;
    if (threadIdx.x < 16) tab[threadIdx.x] = kNF4[threadIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = K / 32, pairs = p.N / 2, slices = (K + kNf4SliceK - 1) / kNf4SliceK;
    const size_t row_chunks = static_cast<size_t>(chunks), row_blocks = static_cast<size_t>(K / kNf4Block);
    const int ldo = p.out_ld ? p.out_ld : (MODE == GEMM_BIAS_SWIGLU_SPLIT ? p.N / 2 : p.N);
    const uint4* c4 = reinterpret_cast<const uint4*>(codes);
    // pairs % 64 == 0 (N % 128 == 0): every warp of a CTA runs the same number of iterations, so the block barriers of
    // the staging are reached by all of them
    for (int pi = blockIdx.x * kGemvPairs + warp; pi < pairs; pi += gridDim.x * kGemvPairs) {
        const int r0 = 128 * (pi >> 6) + (pi & 63), r1 = r0 + 64;
        const uint4* c0 = c4 + r0 * row_chunks;
        const uint4* c1 = c4 + r1 * row_chunks;
        const float* a0 = absmax + r0 * row_blocks;
        const float* a1 = absmax + r1 * row_blocks;
        float acc0[MM], acc1[MM];
#pragma unroll
        for (int m = 0; m < MM; ++m) { acc0[m] = 0.f; acc1[m] = 0.f; }
        int ch = lane;
        uint4 u0{}, u1{};
        float s0 = 0.f, s1 = 0.f;
        if (ch < chunks) { u0 = __ldcs(c0 + ch); u1 = __ldcs(c1 + ch); s0 = __ldg(a0 + (ch >> 1)); s1 = __ldg(a1 + (ch >> 1)); }
        for (int sl = 0; sl < slices; ++sl, ch += 32) {
            const int nx = ch + 32;
            uint4 v0{}, v1{};
            float t0 = 0.f, t1 = 0.f;
            if (nx < chunks) { v0 = __ldcs(c0 + nx); v1 = __ldcs(c1 + nx); t0 = __ldg(a0 + (nx >> 1)); t1 = __ldg(a1 + (nx >> 1)); }
            const int k0 = sl * kNf4SliceK, kn = min(kNf4SliceK, K - k0);
            __syncthreads();                                            // the previous slice is consumed
            for (int e = 2 * threadIdx.x; e < M * kNf4SliceK; e += 2 * kGemvThreads) {
                const int m = e / kNf4SliceK, k = e % kNf4SliceK;
                if (k >= kn) continue;
                const size_t o = static_cast<size_t>(m) * K + k0 + k;
                const float2 h = __half22float2(*reinterpret_cast<const __half2*>(x_hi + o));
                const float2 l = __half22float2(*reinterpret_cast<const __half2*>(x_lo + o));
                *reinterpret_cast<float2*>(xs + m * kNf4SliceK + nf4_x_slot(k)) = make_float2(h.x + l.x, h.y + l.y);
            }
            __syncthreads();
            if (ch < chunks) {
                float w0[32], w1[32];
                const uint32_t q0[4] = {u0.x, u0.y, u0.z, u0.w}, q1[4] = {u1.x, u1.y, u1.z, u1.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const unsigned y0 = (q0[j] >> (8 * b)) & 255u, y1 = (q1[j] >> (8 * b)) & 255u;
                        const float2 f0 = __half22float2(__floats2half2_rn(__fmul_rn(tab[y0 >> 4], s0), __fmul_rn(tab[y0 & 15u], s0)));
                        const float2 f1 = __half22float2(__floats2half2_rn(__fmul_rn(tab[y1 >> 4], s1), __fmul_rn(tab[y1 & 15u], s1)));
                        w0[8 * j + 2 * b] = f0.x; w0[8 * j + 2 * b + 1] = f0.y;
                        w1[8 * j + 2 * b] = f1.x; w1[8 * j + 2 * b + 1] = f1.y;
                    }
                }
                const int sw = ch & 7;
#pragma unroll
                for (int m = 0; m < MM; ++m) {
                    if (m >= M) break;
                    const float4* xv = reinterpret_cast<const float4*>(xs + m * kNf4SliceK + 32 * lane);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float4 xa = xv[j ^ sw];
                        const float xx[4] = {xa.x, xa.y, xa.z, xa.w};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            acc0[m] = fmaf(w0[4 * j + i], xx[i], acc0[m]);
                            acc1[m] = fmaf(w1[4 * j + i], xx[i], acc1[m]);
                        }
                    }
                }
            }
            u0 = v0; u1 = v1; s0 = t0; s1 = t1;
        }
#pragma unroll
        for (int m = 0; m < MM; ++m) {
            if (m >= M) break;
            float e0 = acc0[m], e1 = acc1[m];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                e0 += __shfl_xor_sync(0xffffffffu, e0, o);
                e1 += __shfl_xor_sync(0xffffffffu, e1, o);
            }
            if (lane != 0) continue;
            const size_t oo = static_cast<size_t>(m) * ldo;
            if constexpr (MODE == GEMM_BIAS_SWIGLU_SPLIT) {
                const float g = e0 + p.bias[r0];
                const float v = g / (1.0f + expf(-g)) * (e1 + p.bias[r1]);
                __half h, l;
                split_f16(v, h, l);
                p.out_hi[oo + pi] = h;
                p.out_lo[oo + pi] = l;
                if (p.range_flag && !(fabsf(v) <= 65504.0f)) atomicOr(p.range_flag, 1);
            } else {
                float v0 = e0 + p.bias[r0], v1 = e1 + p.bias[r1];
                if constexpr (MODE == GEMM_BIAS_RESF32_F32) {
                    v0 = v0 + p.res_f32[static_cast<size_t>(m) * p.N + r0];
                    v1 = v1 + p.res_f32[static_cast<size_t>(m) * p.N + r1];
                }
                p.out_f32[oo + r0] = v0;
                p.out_f32[oo + r1] = v1;
            }
        }
    }
}

int launch_nf4_quantize(const __half* hi, int64_t n, uint8_t* codes, float* absmax, cudaStream_t st) {
    ProfScope _ps(PROF_NF4, st);
    const int64_t nblocks = n / kNf4Block;
    if (nblocks == 0) return RMU_OK;
    nf4_quantize_kernel<<<static_cast<unsigned>((nblocks + 7) / 8), 256, 0, st>>>(hi, nblocks, codes, absmax);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

int launch_nf4_dequantize(const uint8_t* codes, const float* absmax, int64_t n, __half* hi, cudaStream_t st) {
    ProfScope _ps(PROF_NF4, st);
    const int64_t n8 = n / 8;
    if (n8 == 0) return RMU_OK;
    const int64_t grid = std::min<int64_t>((n8 + 255) / 256, static_cast<int64_t>(device_sm_count()) * 16);
    nf4_dequantize_kernel<<<static_cast<unsigned>(grid), 256, 0, st>>>(reinterpret_cast<const uint32_t*>(codes), absmax,
                                                                        n8, reinterpret_cast<uint4*>(hi));
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

template <int MODE>
static int gemv_mode(const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p, int sms,
                     cudaStream_t st) {
    // the attribute is per device and the call is cheap: set it on every launch (one process may drive several GPUs)
    RMU_CUDA(cudaFuncSetAttribute(nf4_gemv_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  kNf4MaxK * static_cast<int>(sizeof(float))));
    const size_t smem = static_cast<size_t>(p.K) * sizeof(float);
    const int per_sm = std::max(1, std::min<int>(kGemvCtasPerSm, static_cast<int>((227u << 10) / (smem + 1024))));
    const int groups = p.N / (2 * kGemvPairs);
    const int grid = std::min(groups, sms * per_sm);
    nf4_gemv_kernel<MODE><<<grid, kGemvThreads, smem, st>>>(x_hi, x_lo, W.codes, W.absmax, p);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

template <int MODE, int MM>
static int gemv_rows_mode(const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p, int sms,
                          cudaStream_t st) {
    const int smem = p.M * kNf4SliceK * static_cast<int>(sizeof(float));
    RMU_CUDA(cudaFuncSetAttribute(nf4_gemv_rows_kernel<MODE, MM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  kNf4MaxRows * kNf4SliceK * static_cast<int>(sizeof(float))));
    const int groups = p.N / (2 * kGemvPairs);
    const int grid = std::min(groups, sms * gemv_rows_ctas(MM));
    nf4_gemv_rows_kernel<MODE, MM><<<grid, kGemvThreads, smem, st>>>(x_hi, x_lo, p.M, W.codes, W.absmax, p);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

template <int MODE>
static int gemv_rows_width(const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p, int sms,
                           cudaStream_t st) {
    if (p.M <= 4) return gemv_rows_mode<MODE, 4>(x_hi, x_lo, W, p, sms, st);
    if (p.M <= 8) return gemv_rows_mode<MODE, 8>(x_hi, x_lo, W, p, sms, st);
    return gemv_rows_mode<MODE, kNf4MaxRows>(x_hi, x_lo, W, p, sms, st);
}

int launch_nf4_gemv_rows(int mode, const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p,
                         int sms, cudaStream_t st) {
    ProfScope _ps(PROF_NF4, st);
    switch (mode) {
        case GEMM_BIAS_F32: return gemv_rows_width<GEMM_BIAS_F32>(x_hi, x_lo, W, p, sms, st);
        case GEMM_BIAS_RESF32_F32: return gemv_rows_width<GEMM_BIAS_RESF32_F32>(x_hi, x_lo, W, p, sms, st);
        case GEMM_BIAS_SWIGLU_SPLIT: return gemv_rows_width<GEMM_BIAS_SWIGLU_SPLIT>(x_hi, x_lo, W, p, sms, st);
        default: set_error("nf4 gemv: mode must be 0, 6 or 7"); return RMU_ERR_UNSUPPORTED;
    }
}

int launch_nf4_gemv(int mode, const __half* x_hi, const __half* x_lo, const Nf4Weight& W, const GemmParams& p, int sms,
                    cudaStream_t st) {
    ProfScope _ps(PROF_NF4, st);
    switch (mode) {
        case GEMM_BIAS_F32: return gemv_mode<GEMM_BIAS_F32>(x_hi, x_lo, W, p, sms, st);
        case GEMM_BIAS_RESF32_F32: return gemv_mode<GEMM_BIAS_RESF32_F32>(x_hi, x_lo, W, p, sms, st);
        case GEMM_BIAS_SWIGLU_SPLIT: return gemv_mode<GEMM_BIAS_SWIGLU_SPLIT>(x_hi, x_lo, W, p, sms, st);
        default: set_error("nf4 gemv: mode must be 0, 6 or 7"); return RMU_ERR_UNSUPPORTED;
    }
}

}  // namespace rmu
