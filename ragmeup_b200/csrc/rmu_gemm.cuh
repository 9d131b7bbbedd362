// fp32-accurate GEMM on the 16-bit tensor path of sm_90a.
//
//   C[M,N] = A[M,K] * W[N,K]^T      (both operands K-major, as nn.Linear stores W)
//
// The reference runs these contractions in fp32 (torch nn.Linear inside transformers' BertModel;
// SURVEY.md H3/H9) and BASELINE.json demands 1e-3 parity on logits, which neither TF32 nor bf16
// operands hold on trained-like weights (measured in DESIGN.md).  Operands are therefore carried as
// SPLIT fp16 PLANES, v = hi + lo with hi = fp16(v), lo = fp16(v - hi) (22 mantissa bits), and each
// K step issues three wgmma f16 MMAs: hi*hi + lo*hi + hi*lo, fp32 accumulate in registers.
//
// 128x128 output tiles, K blocks of 64 (one 128-byte swizzled row per operand row), 3-stage smem ring
// (4 planes x 16 KB per stage) filled by TMA.
//
// E1 (gemm_f16x3_kernel) is persistent and PING-PONG scheduled: 1 CTA/SM, 384 threads = one producer
// warpgroup (one elected lane issues the TMA loads, 40 registers per thread) + two consumer warpgroups
// (232 registers per thread).  Each consumer warpgroup owns a whole tile (128 fp32 accumulators per
// thread); consecutive tiles of a CTA alternate between the two.  A pair of named barriers hands the
// tensor cores from one warpgroup to the other once all MMAs of a tile are issued, so one warpgroup
// issues its MMAs while the other runs its epilogue (bias / GELU / split / residual and the TMA stores);
// with K = 384 the mainloop is only 6 K blocks, so without the overlap the epilogue stalls the tensor cores.
// The producer fills the ring in tile order; every consumer warpgroup steps its ring slot and phase past
// the other warpgroup's K blocks.  The ordering barrier also keeps a warpgroup from waiting on a stage
// whose barrier is more than one phase behind (the parity test would alias).
#pragma once
#include "rmu_common.h"
#include "rmu_ptx.cuh"

namespace rmu {

constexpr int kGemmBM = 128, kGemmBN = 128, kGemmBK = 64;
constexpr int kGemmStages = 3;
constexpr int kGemmPlaneBytes = 128 * 128;                 // one plane of a stage: 128 rows x 128 B
constexpr int kGemmStageBytes = 4 * kGemmPlaneBytes;       // A hi | A lo | W hi | W lo
constexpr int kGemmThreads = 3 * 128;                      // E1: producer warpgroup + two consumer warpgroups
constexpr int kGemmProducerRegs = 40, kGemmConsumerRegs = 232;
static_assert(128 * kGemmProducerRegs + 256 * kGemmConsumerRegs <= 65536, "register file");
constexpr int kGemmOrderBar = 1;                           // named barriers 1, 2: "warpgroup w may issue its MMAs"
constexpr int kGemmEpiBar = 3;                             // named barriers 3, 4: warpgroup w's staging buffer
constexpr int kGemmStagingBytes = 128 * 128;               // per consumer warpgroup: one 128-row x 128-byte output box
constexpr size_t kGemmSmem = static_cast<size_t>(kGemmStages) * kGemmStageBytes + 2 * kGemmStagingBytes + 256 + 1024;
static_assert(kGemmSmem <= 232448, "shared memory budget");

enum GemmMode {
    GEMM_BIAS_F32 = 0,        // out_f32 = acc + bias
    GEMM_BIAS_GELU_SPLIT = 1, // out planes = split(gelu_erf(acc + bias))
    GEMM_BIAS_RESID_F32 = 2,  // out_f32 = acc + bias + (res_hi + res_lo)
    GEMM_BIAS_SPLIT_QSCALE = 3, // out planes = split((acc + bias) * (col < qcols ? qscale : 1))   (QKV projection)
    // ModernBERT (pre-LN, rotary positions, GeGLU):
    GEMM_BIAS_SPLIT_ROPE = 4,   // GEMM_BIAS_SPLIT_QSCALE with the q and k columns (col < 2 qcols) rotated per head at the
                                // row's position: x'[c] = x[c] cos - x[c + d/2] sin, x'[c + d/2] = x[c + d/2] cos + x[c] sin
    GEMM_BIAS_GEGLU_SPLIT = 5,  // W's rows in 128-row blocks of 64 input rows | the 64 matching gate rows: out planes
                                // [M, N / 2] = split(gelu_erf(in + b_in) * (gate + b_gate))
    GEMM_BIAS_RESF32_F32 = 6,   // out_f32 = acc + bias + res_f32 (res_f32 may be out_f32: in place)
    // Qwen3 (SwiGLU):
    GEMM_BIAS_SWIGLU_SPLIT = 7, // GEMM_BIAS_GEGLU_SPLIT's row blocks with silu in place of gelu: out planes [M, N / 2] =
                                // split(silu(in + b_in) * (gate + b_gate)); an output row < M with |x| > 65504 (or
                                // NaN) sets *range_flag when it is non-null
};
// the modes whose W holds 64-row input | gate blocks and whose tiles write 64 output columns
__host__ __device__ constexpr bool gemm_gated(int mode) { return mode == GEMM_BIAS_GEGLU_SPLIT || mode == GEMM_BIAS_SWIGLU_SPLIT; }

struct GemmParams {
    int M, N, K;
    const float* bias;                    // [N]
    float* out_f32;                       // [M, N]
    __half* out_hi; __half* out_lo;       // [M, N]
    const __half* res_hi; const __half* res_lo;  // [M, N]
    int qcols; float qscale;              // GEMM_BIAS_SPLIT_QSCALE
    int out_ld;                           // row pitch of out_f32 / out_hi / out_lo in elements (0 = N)
    // (appended, so the fields above keep their offsets)
    const float* res_f32;                 // [M, N] GEMM_BIAS_RESF32_F32
    const int* pos;                       // [M] GEMM_BIAS_SPLIT_ROPE: each row's position within its sequence
    const float* rope_cos; const float* rope_sin;   // [rope_rows, rope_hd / 2] fp32 tables
    int rope_hd, rope_rows;               // head dim (32 or 64) and the tables' rows (positions clamp into them)
    int* range_flag;                      // GEMM_BIAS_SWIGLU_SPLIT: set to 1 when an output leaves the fp16 range
};

__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

// erf by Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, the fp32 noise floor of the erf-GELU the
// reference computes with torch.erf) on the fast exp / reciprocal units: the FFN-in epilogue is ALU-bound.
__device__ __forceinline__ float erf_as(float x) {
    const float ax = fabsf(x);
    const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
    float p = fmaf(1.061405429f, t, -1.453152027f);
    p = fmaf(p, t, 1.421413741f);
    p = fmaf(p, t, -0.284496736f);
    p = fmaf(p, t, 0.254829592f);
    const float y = 1.0f - p * t * __expf(-ax * ax);
    return copysignf(y, x);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752440f)); }

// (a, b) -> fp16 pair of the high parts and fp16 pair of the residuals
__device__ __forceinline__ void split_f16x2(float2 v, __half2& hi, __half2& lo) {
    hi = __floats2half2_rn(v.x, v.y);
    const float2 h = __half22float2(hi);
    lo = __floats2half2_rn(v.x - h.x, v.y - h.y);
}

// TMA producer (one elected lane of the producer warp): the 4 planes of every K block of `tiles` row / column tiles
__device__ __forceinline__ void gemm_produce(uint8_t* smem, uint64_t* full, uint64_t* empty, const CUtensorMap* tAh,
                                             const CUtensorMap* tAl, const CUtensorMap* tWh, const CUtensorMap* tWl,
                                             int mb, int nb, int k_blks, int& slot, uint32_t& phase) {
    for (int kb = 0; kb < k_blks; ++kb) {
        mbar_wait(&empty[slot], phase ^ 1);
        uint8_t* st = smem + slot * kGemmStageBytes;
        mbar_arrive_expect_tx(&full[slot], kGemmStageBytes);
        tma_load_2d(st, tAh, kb * kGemmBK, mb * kGemmBM, &full[slot], kEvictNormal);
        tma_load_2d(st + kGemmPlaneBytes, tAl, kb * kGemmBK, mb * kGemmBM, &full[slot], kEvictNormal);
        tma_load_2d(st + 2 * kGemmPlaneBytes, tWh, kb * kGemmBK, nb * kGemmBN, &full[slot], kEvictLast);
        tma_load_2d(st + 3 * kGemmPlaneBytes, tWl, kb * kGemmBK, nb * kGemmBN, &full[slot], kEvictLast);
        if (++slot == kGemmStages) { slot = 0; phase ^= 1; }
    }
}

__device__ __forceinline__ void ring_advance(int& slot, uint32_t& phase, int n) {
    for (int i = 0; i < n; ++i)
        if (++slot == kGemmStages) { slot = 0; phase ^= 1; }
}

// E1 consumer warpgroup: acc0 / acc1 = rows 0..63 / 64..127 of the tile, each the sum over K of the three split
// products (per element: K steps in order, hi*hi, lo*hi, hi*lo).  One MMA group stays in flight: the slot of the
// previous K block is handed back (one arrive per warp) once its group has retired.  Returns with the last group still
// in flight; the caller retires it (wgmma_wait<0>) and hands back the returned slot.
__device__ __forceinline__ int gemm_mainloop_tile(float (&acc0)[64], float (&acc1)[64], uint8_t* smem, uint64_t* full,
                                                  uint64_t* empty, int k_blks, int& slot, uint32_t& phase) {
    const unsigned lane = lane_id();
    int prev = -1;
    for (int kb = 0; kb < k_blks; ++kb) {
        mbar_wait(&full[slot], phase);
        const uint32_t sbase = smem_u32(smem + slot * kGemmStageBytes);
        const uint64_t dAh0 = wgmma_desc_sw128(sbase);
        const uint64_t dAh1 = wgmma_desc_sw128(sbase + 64 * 128);
        const uint64_t dAl0 = wgmma_desc_sw128(sbase + kGemmPlaneBytes);
        const uint64_t dAl1 = wgmma_desc_sw128(sbase + kGemmPlaneBytes + 64 * 128);
        const uint64_t dWh = wgmma_desc_sw128(sbase + 2 * kGemmPlaneBytes);
        const uint64_t dWl = wgmma_desc_sw128(sbase + 3 * kGemmPlaneBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBK / 16; ++k) {
            const uint64_t off = static_cast<uint64_t>(k * 2);   // 16 halves = 32 B = 2 x 16 B units
            const uint32_t accum = (kb | k) != 0 ? 1u : 0u;
            wgmma_f16_n128(acc0, dAh0 + off, dWh + off, accum);
            wgmma_f16_n128(acc1, dAh1 + off, dWh + off, accum);
            wgmma_f16_n128(acc0, dAl0 + off, dWh + off, 1u);
            wgmma_f16_n128(acc1, dAl1 + off, dWh + off, 1u);
            wgmma_f16_n128(acc0, dAh0 + off, dWl + off, 1u);
            wgmma_f16_n128(acc1, dAh1 + off, dWl + off, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
        prev = slot;
        ring_advance(slot, phase, 1);
    }
    return prev;
}

// GEMM_BIAS_SPLIT_ROPE's values of one 64-column block (block c of the tile, first column col0) -> w (hi pair, lo pair).
// The block is one head (d_h = 64) or two (d_h = 32); HALF8 = d_h / 16 is the distance, in 8-column groups, between the
// two columns of a rotated pair, so both live in this thread (groups j and j + HALF8) and every index is static.  The
// rotated values replace the accumulators of the block (which nothing reads afterwards), so no more registers are live
// than in the other split modes.
template <int HALF8>
__device__ __forceinline__ void rope_rotate(float (&acc)[2][64], const GemmParams& p, int row0, int c, int csub) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int grow = row0 + r * 64 + 8 * h;
            int ps = grow < p.M ? __ldg(p.pos + grow) : 0;
            ps = ps < 0 ? 0 : (ps >= p.rope_rows ? p.rope_rows - 1 : ps);
            const float* ct = p.rope_cos + static_cast<size_t>(ps) * (HALF8 * 8);
            const float* st = p.rope_sin + static_cast<size_t>(ps) * (HALF8 * 8);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                if ((jj / HALF8) % 2 != 0) continue;                 // the second half of a head: rotated with its partner
                const int i = 8 * (jj % HALF8) + csub;               // frequency index of columns (i, i + 1)
                const float2 cs = __ldg(reinterpret_cast<const float2*>(ct + i));
                const float2 sn = __ldg(reinterpret_cast<const float2*>(st + i));
                float* a = &acc[r][4 * (8 * c + jj) + 2 * h];
                float* b = &acc[r][4 * (8 * c + jj + HALF8) + 2 * h];
                const float a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
                a[0] = a0 * cs.x - b0 * sn.x; a[1] = a1 * cs.y - b1 * sn.y;
                b[0] = b0 * cs.x + a0 * sn.x; b[1] = b1 * cs.y + a1 * sn.y;
            }
        }
    }
}

__device__ __forceinline__ void rope_epilogue(float (&acc)[2][64], uint32_t (&w)[2][2][8][2], const GemmParams& p,
                                              int row0, int col0, int c, int csub) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
        const float2 bia2 = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * jj + csub));
        const int j = 8 * c + jj;
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                acc[r][4 * j + 2 * h] += bia2.x;
                acc[r][4 * j + 2 * h + 1] += bia2.y;
            }
    }
    if (col0 < 2 * p.qcols) {                                        // q and k: rotated; v (col >= 2 qcols) is not
        if (p.rope_hd == 64) rope_rotate<4>(acc, p, row0, c, csub);
        else rope_rotate<2>(acc, p, row0, c, csub);
    }
    const float sc = col0 < p.qcols ? p.qscale : 1.0f;
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int j = 8 * c + jj;
                __half2 h2, l2;
                split_f16x2(make_float2(acc[r][4 * j + 2 * h] * sc, acc[r][4 * j + 2 * h + 1] * sc), h2, l2);
                w[r][h][jj][0] = *reinterpret_cast<const uint32_t*>(&h2);
                w[r][h][jj][1] = *reinterpret_cast<const uint32_t*>(&l2);
            }
}

// Accumulator layout of wgmma m64nN (f32): thread t of the warpgroup holds rows 16 * (t / 32) + (t % 32) / 4 and + 8,
// columns 8 j + 2 (t % 4) + {0, 1} for j < N / 8, as d[4 j + 2 h + e] (h = second row, e = second column).
//
// Epilogue: the output leaves through the warpgroup's 16 KB staging buffer in four 128-row x 128-byte boxes (split modes:
// column half x plane; fp32 modes: column quarter), each written to shared memory in the 128-byte swizzle (conflict-free
// for the accumulator layout) and stored by one TMA bulk store, which writes whole lines and clips the rows past M.
// Direct 4-byte stores from the accumulator layout cover half a 32-byte sector each and took as long as the mainloop.
template <int MODE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_f16x3_kernel(const __grid_constant__ CUtensorMap tAh, const __grid_constant__ CUtensorMap tAl,
                  const __grid_constant__ CUtensorMap tWh, const __grid_constant__ CUtensorMap tWl,
                  const __grid_constant__ CUtensorMap tOa, const __grid_constant__ CUtensorMap tOb,
                  const GemmParams p) {
    constexpr bool kF32Out = MODE == GEMM_BIAS_F32 || MODE == GEMM_BIAS_RESID_F32 || MODE == GEMM_BIAS_RESF32_F32;
    constexpr int kJB = kF32Out ? 4 : 8;                       // 8-column groups per 128-byte box row
    constexpr int kBoxes = gemm_gated(MODE) ? 1 : kGemmBN / 8 / kJB;   // GeGLU / SwiGLU: 64 output columns per tile
    extern __shared__ uint8_t gemm_smem_raw[];
    // 1024-byte alignment by OFFSET into the shared array (the 128-byte swizzle repeats every 1024 B)
    uint8_t* smem = gemm_smem_raw + ((1024u - (smem_u32(gemm_smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kGemmStages * kGemmStageBytes + 2 * kGemmStagingBytes);
    uint64_t* empty = full + kGemmStages;

    const int warp = threadIdx.x >> 5;
    const unsigned lane = lane_id();
    if (threadIdx.x == 0) {
        for (int i = 0; i < kGemmStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }   // 4 warps release
        fence_mbar_init();
        prefetch_tmap(&tAh); prefetch_tmap(&tAl); prefetch_tmap(&tWh); prefetch_tmap(&tWl);
        prefetch_tmap(&tOa);
        if (!kF32Out) prefetch_tmap(&tOb);
    }
    __syncthreads();

    const int n_blks = p.N / kGemmBN;
    const int k_blks = p.K / kGemmBK;
    const int tiles = ((p.M + kGemmBM - 1) / kGemmBM) * n_blks;
    const int my_tiles = tiles > static_cast<int>(blockIdx.x) ? (tiles - 1 - static_cast<int>(blockIdx.x)) / gridDim.x + 1 : 0;
    int slot = 0;
    uint32_t phase = 0;

    if (warp < 4) {
        setmaxnreg_dec<kGemmProducerRegs>();
        if (warp == 0 && elect_one())
            for (int t = 0; t < my_tiles; ++t) {
                const int tile = blockIdx.x + t * gridDim.x;
                gemm_produce(smem, full, empty, &tAh, &tAl, &tWh, &tWl, tile / n_blks, tile % n_blks, k_blks, slot, phase);
            }
        return;
    }
    setmaxnreg_inc<kGemmConsumerRegs>();

    const int wg = (warp >> 2) - 1;                                    // consumer warpgroup 0 / 1: local tiles wg, wg + 2, ..
    const bool store_lead = (threadIdx.x & 127) == 0;                  // issues the warpgroup's TMA stores and waits for them
    uint8_t* staging = smem + kGemmStages * kGemmStageBytes + wg * kGemmStagingBytes;
    const uint32_t staging_u32 = smem_u32(staging);
    const int rsub = (warp & 3) * 16 + static_cast<int>(lane >> 2);     // first of this thread's two rows in each 64
    const int q4 = static_cast<int>(lane & 3);
    const int csub = 2 * q4;                                           // first of its column pairs in every 8 columns
    ring_advance(slot, phase, wg * k_blks);
    for (int t = wg; t < my_tiles; t += 2) {
        const int tile = blockIdx.x + t * gridDim.x;
        const int mb = tile / n_blks, nb = tile % n_blks;
        float acc[2][64];
        if (t > 0) bar_sync_named(kGemmOrderBar + wg, 256);           // the other warpgroup has issued tile t - 1
        const int last = gemm_mainloop_tile(acc[0], acc[1], smem, full, empty, k_blks, slot, phase);
        // every MMA of this tile is issued: the other warpgroup may queue its own behind them
        if (t + 1 < my_tiles) bar_arrive_named(kGemmOrderBar + (wg ^ 1), 256);
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[last]);
        ring_advance(slot, phase, k_blks);                             // the other warpgroup's tile t + 1
        // ---- epilogue per column block of 32 (fp32) / 64 (split) columns: values into registers, then one 128-row x
        // 128-byte box per output plane through the staging buffer
#pragma unroll
        for (int c = 0; c < kBoxes; ++c) {
            uint32_t w[2][2][kJB][2];                                  // [r][h][jj]: fp32 (x, y) or (hi pair, lo pair)
            if constexpr (MODE == GEMM_BIAS_SPLIT_ROPE) {
                rope_epilogue(acc, w, p, mb * kGemmBM + rsub, nb * kGemmBN + 64 * c, c, csub);
            } else if constexpr (gemm_gated(MODE)) {
                // columns 8 jj + csub of the block are inputs, 64 + 8 jj + csub their gates: both in this thread
#pragma unroll
                for (int r = 0; r < 2; ++r) {
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int col = nb * kGemmBN + 8 * jj + csub;
                        const float2 bi = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                        const float2 bg = __ldg(reinterpret_cast<const float2*>(p.bias + col + 64));
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float2 v;
                            if constexpr (MODE == GEMM_BIAS_SWIGLU_SPLIT) {
                                const float g0 = acc[r][4 * jj + 2 * h] + bi.x, g1 = acc[r][4 * jj + 2 * h + 1] + bi.y;
                                v = make_float2(g0 / (1.0f + expf(-g0)) * (acc[r][4 * (jj + 8) + 2 * h] + bg.x),
                                                g1 / (1.0f + expf(-g1)) * (acc[r][4 * (jj + 8) + 2 * h + 1] + bg.y));
                                // rows past M hold whatever the A rows past M made (the TMA store clips them): not checked
                                const int grow = mb * kGemmBM + r * 64 + rsub + 8 * h;
                                if (p.range_flag && grow < p.M && !(fabsf(v.x) <= 65504.0f && fabsf(v.y) <= 65504.0f))
                                    atomicOr(p.range_flag, 1);
                            } else {
                                v = make_float2(gelu_erf(acc[r][4 * jj + 2 * h] + bi.x) * (acc[r][4 * (jj + 8) + 2 * h] + bg.x),
                                                gelu_erf(acc[r][4 * jj + 2 * h + 1] + bi.y) * (acc[r][4 * (jj + 8) + 2 * h + 1] + bg.y));
                            }
                            __half2 h2, l2;
                            split_f16x2(v, h2, l2);
                            w[r][h][jj][0] = *reinterpret_cast<const uint32_t*>(&h2);
                            w[r][h][jj][1] = *reinterpret_cast<const uint32_t*>(&l2);
                        }
                    }
                }
            } else {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
#pragma unroll
                for (int jj = 0; jj < kJB; ++jj) {
                    const int j = kJB * c + jj;
                    const int col = nb * kGemmBN + 8 * j + csub;
                    const float2 bia2 = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                    const float sc = (MODE == GEMM_BIAS_SPLIT_QSCALE && col < p.qcols) ? p.qscale : 1.0f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int grow = mb * kGemmBM + r * 64 + rsub + 8 * h;
                        float2 v = make_float2(acc[r][4 * j + 2 * h] + bia2.x, acc[r][4 * j + 2 * h + 1] + bia2.y);
                        if (MODE == GEMM_BIAS_GELU_SPLIT) v = make_float2(gelu_erf(v.x), gelu_erf(v.y));
                        if (MODE == GEMM_BIAS_SPLIT_QSCALE) v = make_float2(v.x * sc, v.y * sc);
                        if (MODE == GEMM_BIAS_RESID_F32 && grow < p.M) {
                            const size_t o = static_cast<size_t>(grow) * p.N + col;
                            const float2 rh = __half22float2(*reinterpret_cast<const __half2*>(p.res_hi + o));
                            const float2 rl = __half22float2(*reinterpret_cast<const __half2*>(p.res_lo + o));
                            v = make_float2(v.x + (rh.x + rl.x), v.y + (rh.y + rl.y));
                        }
                        if (MODE == GEMM_BIAS_RESF32_F32 && grow < p.M) {
                            const float2 rr = *reinterpret_cast<const float2*>(p.res_f32 + static_cast<size_t>(grow) * p.N + col);
                            v = make_float2(v.x + rr.x, v.y + rr.y);
                        }
                        if (kF32Out) {
                            w[r][h][jj][0] = __float_as_uint(v.x);
                            w[r][h][jj][1] = __float_as_uint(v.y);
                        } else {
                            __half2 h2, l2;
                            split_f16x2(v, h2, l2);
                            w[r][h][jj][0] = *reinterpret_cast<const uint32_t*>(&h2);
                            w[r][h][jj][1] = *reinterpret_cast<const uint32_t*>(&l2);
                        }
                    }
                }
            }
            }
#pragma unroll
            for (int pl = 0; pl < (kF32Out ? 1 : 2); ++pl) {
                if (store_lead) bulk_wait_read<0>();                  // the previous box has left the staging buffer
                bar_sync_named(kGemmEpiBar + wg, 128);
#pragma unroll
                for (int r = 0; r < 2; ++r) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r * 64 + rsub + 8 * h;
                        const uint32_t rbase = staging_u32 + row * 128;   // 16-byte chunk k of the row lives at k ^ (row & 7)
                        const int sw = row & 7;
#pragma unroll
                        for (int jj = 0; jj < kJB; ++jj) {
                            if (kF32Out) st_shared_v2(rbase + (((2 * jj + (q4 >> 1)) ^ sw) << 4) + 8 * (q4 & 1), w[r][h][jj][0], w[r][h][jj][1]);
                            else st_shared_b32(rbase + ((jj ^ sw) << 4) + 4 * q4, w[r][h][jj][pl]);
                        }
                    }
                }
                fence_proxy_async_smem();                              // generic-proxy writes -> visible to the TMA store
                bar_sync_named(kGemmEpiBar + wg, 128);
                if (store_lead) {
                    tma_store_2d(pl ? &tOb : &tOa, staging, gemm_gated(MODE) ? nb * 64 : nb * kGemmBN + 8 * kJB * c,
                                 mb * kGemmBM);
                    bulk_commit();
                }
            }
        }
    }
    if (store_lead) bulk_wait<0>();                                    // the stores have completed before the CTA retires
}

// A K-major fp16 operand carried as two planes, with the TMA maps of both (box {64 halves, 128 rows}, SWIZZLE_128B)
struct SplitOperand {
    __half* hi = nullptr;
    __half* lo = nullptr;
    int64_t rows = 0;     // rows covered by the tensor maps (allocation rows)
    int cols = 0;
    CUtensorMap map_hi{}, map_lo{};
};

int make_split_operand(SplitOperand* op, __half* hi, __half* lo, int64_t rows, int cols);
// C = A * W^T with the epilogue `mode`; A rows used = p.M (<= A.rows)
int launch_gemm(int mode, const SplitOperand& A, const SplitOperand& W, const GemmParams& p, int sms, cudaStream_t st);

}  // namespace rmu
