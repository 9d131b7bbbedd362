// Post-LN BERT encoder forward for sm_90a: sentence embeddings and cross-encoder logits.
//
// Stands behind HuggingFaceEmbeddings.embed_documents / embed_query (reference call sites
// server/RAGHelper_local.py:114-117, server/RAGHelper_cloud.py:101-103; arithmetic = transformers
// BertModel + sentence-transformers Pooling/Normalize, SURVEY.md H2-H4) and behind
// HuggingFaceCrossEncoder.score (server/RAGHelper.py:484, server/ScoredCrossEncoderReranker.py:42;
// BertForSequenceClassification, H8-H9).  SURVEY.md §8 rows a2-a5, a9, a10.
//
// Batches are RAGGED (cu_seqlens): no padding token is ever computed.  The reference pads to the
// longest sequence of each 32-batch and masks padded keys with finfo.min, which contributes exactly
// 0 to every softmax, so the packed computation returns the same numbers.
//
// Activations between kernels are split fp16 planes (see rmu_gemm.cuh); LayerNorm, softmax, GELU,
// residual adds, pooling and the classifier head are fp32.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <type_traits>
#include <vector>

#include "rmu_gemm.cuh"
#include "rmu_nf4.cuh"

namespace rmu {

// ------------------------------------------------------------------------------------ small kernels
__global__ void split_planes_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, size_t n) {
    size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) {
        __half h, l;
        split_f16(src[i], h, l);
        hi[i] = h;
        lo[i] = l;
    }
}

constexpr int kMaxPerLane = 32;  // hidden <= 1024

// LayerNorm of one row (H % 128 == 0).  Lane l holds float4 chunks l, l + 32, l + 64 ... of the row
// (element v[i] is column ((i / 4) * 32 + l) * 4 + i % 4), so every warp load is one contiguous 512-byte
// segment and every plane store one contiguous 256-byte segment.  Biased variance, eps inside the sqrt
// (nn.LayerNorm).
__device__ __forceinline__ void warp_layernorm_store(float (&v)[kMaxPerLane], int per_lane, int H, float eps,
                                                     const float* __restrict__ g, const float* __restrict__ b,
                                                     __half* __restrict__ hi, __half* __restrict__ lo) {
    const unsigned lane = lane_id();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) if (i < per_lane) s += v[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / static_cast<float>(H);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) if (i < per_lane) { const float d = v[i] - mean; q = fmaf(d, d, q); }
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.0f / sqrtf(q / static_cast<float>(H) + eps);
#pragma unroll
    for (int i = 0; i < kMaxPerLane; i += 4) {
        if (i < per_lane) {
            const int col = (i * 8 + static_cast<int>(lane)) * 4;      // (i / 4) * 32 + lane, in float4 units
            const float4 gg = *reinterpret_cast<const float4*>(g + col);
            const float4 bb = *reinterpret_cast<const float4*>(b + col);
            const float y0 = (v[i] - mean) * rstd * gg.x + bb.x, y1 = (v[i + 1] - mean) * rstd * gg.y + bb.y;
            const float y2 = (v[i + 2] - mean) * rstd * gg.z + bb.z, y3 = (v[i + 3] - mean) * rstd * gg.w + bb.w;
            __half h0, l0, h1, l1, h2, l2, h3, l3;
            split_f16(y0, h0, l0); split_f16(y1, h1, l1); split_f16(y2, h2, l2); split_f16(y3, h3, l3);
            __half2 ha = __halves2half2(h0, h1), hb = __halves2half2(h2, h3);
            __half2 la = __halves2half2(l0, l1), lb = __halves2half2(l2, l3);
            uint2 ph, pl;
            ph.x = *reinterpret_cast<uint32_t*>(&ha); ph.y = *reinterpret_cast<uint32_t*>(&hb);
            pl.x = *reinterpret_cast<uint32_t*>(&la); pl.y = *reinterpret_cast<uint32_t*>(&lb);
            *reinterpret_cast<uint2*>(hi + col) = ph;
            *reinterpret_cast<uint2*>(lo + col) = pl;
        }
    }
}

// word + position + token-type embedding sum -> LayerNorm -> split planes.  One warp per token.
// POS = RMU_POS_OFFSET (MPNet, RoBERTa): HF's create_position_ids_from_input_ids with padding_idx 1, i.e. a token of
// id 1 takes position 1 and any other token at offset j takes 2 + j - (tokens of id 1 before it).  The warp counts those
// with one ballot per 32 tokens of the prefix.  POS = RMU_POS_ABSOLUTE (BERT) is position j.
constexpr int kPadId = 1;
template <int POS>
__global__ void embed_ln_kernel(const int* __restrict__ ids, const int* __restrict__ type_ids,
                                const int* __restrict__ cu, int B, int T, int H, int vocab, int max_pos, int type_vocab,
                                const float* __restrict__ word, const float* __restrict__ pos,
                                const float* __restrict__ typ, const float* __restrict__ g, const float* __restrict__ b,
                                float eps, __half* __restrict__ hi, __half* __restrict__ lo) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= T) return;
    // sequence of token t: last b with cu[b] <= t
    int lo_b = 0, hi_b = B;
    while (hi_b - lo_b > 1) {
        const int mid = (lo_b + hi_b) >> 1;
        if (cu[mid] <= t) lo_b = mid; else hi_b = mid;
    }
    int p = t - cu[lo_b];
    if constexpr (POS == RMU_POS_OFFSET) {
        const int* seq = ids + cu[lo_b];
        int pads = 0;
        for (int k0 = 0; k0 < p; k0 += 32) {
            const int k = k0 + static_cast<int>(lane_id());
            pads += __popc(__ballot_sync(0xffffffffu, k < p && seq[k] == kPadId));
        }
        p = ids[t] == kPadId ? kPadId : p + kPadId + 1 - pads;
    }
    p = p < max_pos ? p : max_pos - 1;
    int id = ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    int ty = type_ids ? type_ids[t] : 0;
    ty = ty < 0 ? 0 : (ty >= type_vocab ? type_vocab - 1 : ty);
    const int per_lane = H >> 5;
    const int l4 = static_cast<int>(lane_id()) * 4;
    const float* w = word + static_cast<size_t>(id) * H + l4;
    const float* pp = pos + static_cast<size_t>(p) * H + l4;
    const float* tt = typ + static_cast<size_t>(ty) * H + l4;
    float v[kMaxPerLane];
#pragma unroll
    for (int i = 0; i < kMaxPerLane; i += 4) {
        if (i < per_lane) {
            const float4 a = *reinterpret_cast<const float4*>(w + i * 32);
            const float4 c = *reinterpret_cast<const float4*>(tt + i * 32);
            const float4 e = *reinterpret_cast<const float4*>(pp + i * 32);
            // HF: inputs_embeds + token_type_embeddings, then + position_embeddings
            v[i] = (a.x + c.x) + e.x; v[i + 1] = (a.y + c.y) + e.y; v[i + 2] = (a.z + c.z) + e.z; v[i + 3] = (a.w + c.w) + e.w;
        }
    }
    warp_layernorm_store(v, per_lane, H, eps, g, b, hi + static_cast<size_t>(t) * H, lo + static_cast<size_t>(t) * H);
}

// LayerNorm(pre) -> split planes.  One warp per token.
__global__ void ln_kernel(const float* __restrict__ pre, int T, int H, const float* __restrict__ g,
                          const float* __restrict__ b, float eps, __half* __restrict__ hi, __half* __restrict__ lo) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= T) return;
    const int per_lane = H >> 5;
    const float* row = pre + static_cast<size_t>(t) * H + lane_id() * 4;
    float v[kMaxPerLane];
#pragma unroll
    for (int i = 0; i < kMaxPerLane; i += 4) {
        if (i < per_lane) {
            const float4 a = *reinterpret_cast<const float4*>(row + i * 32);
            v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
        }
    }
    warp_layernorm_store(v, per_lane, H, eps, g, b, hi + static_cast<size_t>(t) * H, lo + static_cast<size_t>(t) * H);
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void split_pack(float x, float y, uint32_t& hi, uint32_t& lo) {
    __half hx, lx, hy, ly;
    split_f16(x, hx, lx);
    split_f16(y, hy, ly);
    __half2 h = __halves2half2(hx, hy), l = __halves2half2(lx, ly);
    hi = *reinterpret_cast<uint32_t*>(&h);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

constexpr int kKeySB = 256;   // keys resident in shared memory at a time

// ---------------------------------------------------------------------------------------------------
// attention_planes_kernel (mma.sync m16n8k16, fp32 accumulate): Q (pre-scaled), K and V arrive as
// split fp16 planes [T, 3H] written by the QKV GEMM epilogue, so this kernel does no conversion work:
// K / V tiles are 16-byte copies into shared memory ([key][d] for both) and the P V operand is fetched
// with ldmatrix.trans.  One CTA = (sequence, head, block of 16*NW query rows), one warp = 16 rows.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_row)));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_row)));
}

constexpr int kAttWarps = 10;   // 160 query rows per CTA (a 147-token rerank pair fits one CTA)

__device__ __forceinline__ float fast_exp2(float x) {   // ex2.approx: 2 ulp, exp2(-inf) = +0
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// MINB = CTAs per SM the register allocation is bounded for (d_h = 32: 2 -> 95 registers, no spills; bounding it
// to 3 CTAs / 64 registers spills in the key loop and measured 541 us instead of 352 us per layer call).
// Grid = (heads, sequences, row blocks): the heads of one sequence run together, so the 64-byte (d_h = 32)
// K / V row segments of neighbouring heads are fetched from DRAM as whole lines.
//
// CLS = true: query row 0 of each sequence only, for the last layer when only the CLS rows leave the encoder.  Q comes
// from row b of the compact planes cls_q [B, H], the context goes to row b of ctx [B, H] (zeros for an empty sequence),
// grid z = 1.  Warp 0 runs the same code as warp 0 of the full kernel with query rows 1..15 zero; the MMA rows and the
// softmax rows are independent, so row 0 comes out bit-identical.  The other NW - 1 warps only help stage K / V.
//
// RelBias = const float* (MPNet): the kernel takes one more parameter, rel_bias, and score(i, j) +=
// rel_bias[h][clamp(j - i, -127, 127) + 127], a [heads, kRelSpan] fp32 table already multiplied by log2(e)
// (build_relative_bias_table), with i and j the query and key rows within the sequence.  The CTA's head row of the
// table sits in shared memory behind the V planes.  With the pack empty (BERT) the parameter list and the code are
// those of the kernel without the bias: one more kernel parameter alone changes ptxas's register allocation.
//
// RelBias = KeyLimit (ColBERT queries): the kernel takes nkeys, and sequence b's keys stop at row
// min(max(nkeys[b], 1), S_b) of the sequence.  Every query row still runs; keys at or past the limit are never staged and
// are masked like keys past the sequence end, so with nkeys[b] = S_b the arithmetic is the kernel's without the limit.
struct KeyLimit {
    const int* __restrict__ n;                // [B] keys per sequence, offset by the slice start like cu
};
// RelBias = Disentangled (DeBERTa-v2): score(i, j) += C2P[qrow, h, c] + P2C[t0 + j, h, c] with c = cidx[i - j + rmax] - c0,
// the position terms of launch_position_terms, already in the log2 units of the scores.  qrow is t0 + i, or (CLS) row b
// of the compact C2P rows.  Reads of query rows and keys past the sequence end are clamped into it; those scores are
// discarded or masked as without the terms.
struct Disentangled {
    const float* __restrict__ c2p;            // [rows, heads, W]: the query rows (tokens, or CLS rows offset by the slice)
    const float* __restrict__ p2c;            // [T, heads, W]: every key row
    const int* __restrict__ cidx;             // [2 rmax + 1]: clamp(s + bucket(r), 0, 2s - 1) at r + rmax, r = i - j
    int rmax, c0, W;
};
// RelBias = Window (ModernBERT's local layers, full mode): key j is visible to query i iff |i - j| <= w.  A CTA stages
// only the keys [max(0, rbase - w), min(S, rbase + 16 NW + w)), a warp skips the 32-key blocks outside its rows' windows,
// and the remaining scores outside the window are masked to -inf.  A row can then meet a block whose keys are all masked
// before any visible key: its running max is still -inf, and exp2(-inf - -inf) would be NaN, so (as FlashAttention
// does) the exponent base is 0 while the max is -inf.  With w >= S - 1 the staged keys, their order and every score are
// those of the kernel without the pack, so the output is bit-identical to it.
struct Window {
    int w;
};
template <typename... P> constexpr bool kHasBias = (std::is_same_v<P, const float*> || ...);
template <typename... P> constexpr bool kHasKeyLimit = (std::is_same_v<P, KeyLimit> || ...);
template <typename... P> constexpr bool kHasDis = (std::is_same_v<P, Disentangled> || ...);
template <typename... P> constexpr bool kHasWindow = (std::is_same_v<P, Window> || ...);
constexpr int kRelMax = 127;                  // |j - i| >= 127 all fall in MPNet's last bucket (distance >= 91)
constexpr int kRelSpan = 2 * kRelMax + 1;
template <int DH, int MINB, int NW = kAttWarps, bool CLS = false, typename... RelBias>  // NW warps = 16 * NW query rows per CTA
__global__ void __launch_bounds__(NW * 32, MINB) attention_planes_kernel(const __half* __restrict__ ph, const __half* __restrict__ pl,
                                                                          const __half* __restrict__ cls_q_hi,
                                                                          const __half* __restrict__ cls_q_lo,
                                                                          const int* __restrict__ cu, int H, int ksb,
                                                                          __half* __restrict__ ctx_hi, __half* __restrict__ ctx_lo,
                                                                          RelBias... rel_bias) {
    constexpr int KSTR = DH + 8;
    constexpr int KS = DH / 16;
    constexpr int NT = DH / 8;
    extern __shared__ __align__(16) unsigned char att_smem[];
    __half* Kh = reinterpret_cast<__half*>(att_smem);
    __half* Kl = Kh + ksb * KSTR;           // ksb = keys resident at a time (multiple of 32, <= kKeySB)
    __half* Vh = Kl + ksb * KSTR;
    __half* Vl = Vh + ksb * KSTR;

    const int b = blockIdx.y, h = blockIdx.x;
    const int t0 = cu[b], S = cu[b + 1] - t0;
    if (CLS && S <= 0) {
        for (int c = threadIdx.x; c < DH; c += blockDim.x) {
            ctx_hi[static_cast<size_t>(b) * H + h * DH + c] = __ushort_as_half(0);
            ctx_lo[static_cast<size_t>(b) * H + h * DH + c] = __ushort_as_half(0);
        }
        return;
    }
    const int rbase = blockIdx.z * (NW * 16);
    if (rbase >= S) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const size_t ld = static_cast<size_t>(3) * H;
    // query rows: the sequence's rows of the QKV planes, or (CLS) its one row of the compact Q planes; the context rows
    // start at the same row index, of the [T, H] or the [B, H] output
    const size_t qld = CLS ? static_cast<size_t>(H) : ld;
    const int qrows = CLS ? 1 : S;
    const int orow = CLS ? b : t0;
    const __half* qh_base = CLS ? cls_q_hi + static_cast<size_t>(b) * H + h * DH : ph + static_cast<size_t>(t0) * ld + h * DH;
    const __half* ql_base = CLS ? cls_q_lo + static_cast<size_t>(b) * H + h * DH : pl + static_cast<size_t>(t0) * ld + h * DH;
    const int r0 = rbase + warp * 16;
    const bool warp_live = r0 < qrows;
    if constexpr (kHasBias<RelBias...>) {      // this head's biases, visible after the first __syncthreads of the key loop
        const float* tab = (rel_bias, ...);
        float* relb = reinterpret_cast<float*>(Vl + ksb * KSTR);
        for (int e = threadIdx.x; e < kRelSpan; e += blockDim.x) relb[e] = tab[h * kRelSpan + e];
    }

    uint32_t qh[KS][4], ql[KS][4];
    {
        const int ra = r0 + g, rb = r0 + g + 8;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int i = 0; i < 4; ++i) { qh[ks][i] = 0u; ql[ks][i] = 0u; }
            if (warp_live && ra < qrows) {
                qh[ks][0] = *reinterpret_cast<const uint32_t*>(qh_base + ra * qld + ks * 16 + 2 * t);
                ql[ks][0] = *reinterpret_cast<const uint32_t*>(ql_base + ra * qld + ks * 16 + 2 * t);
                qh[ks][2] = *reinterpret_cast<const uint32_t*>(qh_base + ra * qld + ks * 16 + 2 * t + 8);
                ql[ks][2] = *reinterpret_cast<const uint32_t*>(ql_base + ra * qld + ks * 16 + 2 * t + 8);
            }
            if (warp_live && rb < qrows) {
                qh[ks][1] = *reinterpret_cast<const uint32_t*>(qh_base + rb * qld + ks * 16 + 2 * t);
                ql[ks][1] = *reinterpret_cast<const uint32_t*>(ql_base + rb * qld + ks * 16 + 2 * t);
                qh[ks][3] = *reinterpret_cast<const uint32_t*>(qh_base + rb * qld + ks * 16 + 2 * t + 8);
                ql[ks][3] = *reinterpret_cast<const uint32_t*>(ql_base + rb * qld + ks * 16 + 2 * t + 8);
            }
        }
    }
    float oacc[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) oacc[n][0] = oacc[n][1] = oacc[n][2] = oacc[n][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    // (declared here, next to the key loop: with the block further up, the instantiations without a key limit got
    // another register allocation)
    int SK = S;                                    // keys of this sequence
    if constexpr (kHasKeyLimit<RelBias...>) {
        const KeyLimit lim = (rel_bias, ...);
        SK = min(max(lim.n[b], 1), S);
    }
    int K0 = 0;                                    // first key staged
    if constexpr (kHasWindow<RelBias...>) {
        const Window win = (rel_bias, ...);
        K0 = max(0, rbase - win.w);
        SK = min(S, rbase + NW * 16 + win.w);
    }
    for (int sb0 = K0; sb0 < SK; sb0 += ksb) {
        const int nk = min(ksb, SK - sb0);
        const int nk16 = (nk + 15) & ~15;
        __syncthreads();
        for (int e = threadIdx.x; e < nk16 * (DH / 8); e += blockDim.x) {
            const int j = e / (DH / 8), c8 = (e % (DH / 8)) * 8;
            uint4 kh = make_uint4(0, 0, 0, 0), kl = kh, vh = kh, vl = kh;
            if (j < nk) {
                const size_t o = static_cast<size_t>(t0 + sb0 + j) * ld + h * DH + c8;
                kh = *reinterpret_cast<const uint4*>(ph + o + H);
                kl = *reinterpret_cast<const uint4*>(pl + o + H);
                vh = *reinterpret_cast<const uint4*>(ph + o + 2 * H);
                vl = *reinterpret_cast<const uint4*>(pl + o + 2 * H);
            }
            *reinterpret_cast<uint4*>(Kh + j * KSTR + c8) = kh;
            *reinterpret_cast<uint4*>(Kl + j * KSTR + c8) = kl;
            *reinterpret_cast<uint4*>(Vh + j * KSTR + c8) = vh;
            *reinterpret_cast<uint4*>(Vl + j * KSTR + c8) = vl;
        }
        __syncthreads();
        if (!warp_live) continue;
        for (int kb0 = 0; kb0 < nk16; kb0 += 32) {
            if constexpr (kHasWindow<RelBias...>) {    // every key of the block outside every row's window: no change
                const Window win = (rel_bias, ...);
                const int j0 = sb0 + kb0;
                if (j0 + 31 < r0 - win.w || j0 > r0 + 15 + win.w) continue;
            }
            float sacc[4][4];
#pragma unroll
            for (int n = 0; n < 4; ++n) sacc[n][0] = sacc[n][1] = sacc[n][2] = sacc[n][3] = 0.f;
            const bool full_blk = kb0 + 32 <= nk16;      // else only the first two n-tiles hold keys
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                // K fragments of four key tiles through two ldmatrix.x4 per plane: matrices (keys a, d lo),
                // (keys a, d hi), (keys a+1, d lo), (keys a+1, d hi); rows past nk16 are stale smem, masked below
                uint32_t bh[4][2], bl[4][2];
                const int lrow = (lane & 7) + ((lane >> 4) << 3);
                const int lcol = ks * 16 + ((lane >> 3) & 1) * 8;
#pragma unroll
                for (int n2 = 0; n2 < 2; ++n2) {
                    uint32_t th[4], tl[4];
                    ldmatrix_x4(th, Kh + (kb0 + n2 * 16 + lrow) * KSTR + lcol);
                    ldmatrix_x4(tl, Kl + (kb0 + n2 * 16 + lrow) * KSTR + lcol);
                    bh[2 * n2][0] = th[0]; bh[2 * n2][1] = th[1]; bh[2 * n2 + 1][0] = th[2]; bh[2 * n2 + 1][1] = th[3];
                    bl[2 * n2][0] = tl[0]; bl[2 * n2][1] = tl[1]; bl[2 * n2 + 1][0] = tl[2]; bl[2 * n2 + 1][1] = tl[3];
                }
#pragma unroll
                for (int n = 0; n < 4; ++n) if (n < 2 || full_blk) mma16816(sacc[n], qh[ks], bh[n]);
#pragma unroll
                for (int n = 0; n < 4; ++n) if (n < 2 || full_blk) mma16816(sacc[n], ql[ks], bh[n]);
#pragma unroll
                for (int n = 0; n < 4; ++n) if (n < 2 || full_blk) mma16816(sacc[n], qh[ks], bl[n]);
            }
            if constexpr (kHasBias<RelBias...>) {
                // fragment (n, c): key sb0 + kb0 + n * 8 + 2t + (c & 1), query row r0 + g (c < 2) or r0 + g + 8; keys past
                // the sequence end read a clamped entry and are masked below
                const float* relb = reinterpret_cast<const float*>(Vl + ksb * KSTR);
                const int ja = sb0 + kb0 + 2 * t - (CLS ? 0 : r0 + g);
                const int jb = CLS ? ja : ja - 8;
#pragma unroll
                for (int n = 0; n < 4; ++n) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        sacc[n][c] += relb[min(max(ja + n * 8 + c, -kRelMax), kRelMax) + kRelMax];
                        sacc[n][2 + c] += relb[min(max(jb + n * 8 + c, -kRelMax), kRelMax) + kRelMax];
                    }
                }
            }
            if constexpr (kHasDis<RelBias...>) {
                const Disentangled dis = (rel_bias, ...);
                const size_t rs = static_cast<size_t>(gridDim.x) * dis.W;     // heads * W floats per row
                const int ia = CLS ? 0 : min(r0 + g, S - 1), ib = CLS ? 0 : min(r0 + g + 8, S - 1);
                const float* c2a = dis.c2p + static_cast<size_t>(CLS ? b : t0 + ia) * rs + h * dis.W - dis.c0;
                const float* c2b = dis.c2p + static_cast<size_t>(CLS ? b : t0 + ib) * rs + h * dis.W - dis.c0;
#pragma unroll
                for (int n = 0; n < 4; ++n) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int j = min(sb0 + kb0 + n * 8 + 2 * t + c, S - 1);
                        const float* p2 = dis.p2c + static_cast<size_t>(t0 + j) * rs + h * dis.W - dis.c0;
                        const int ca = __ldg(dis.cidx + ia - j + dis.rmax), cb = __ldg(dis.cidx + ib - j + dis.rmax);
                        sacc[n][c] += __ldg(c2a + ca) + __ldg(p2 + ca);
                        sacc[n][2 + c] += __ldg(c2b + cb) + __ldg(p2 + cb);
                    }
                }
            }
            if constexpr (kHasWindow<RelBias...>) {
                const Window win = (rel_bias, ...);
                const int ia = r0 + g, ib = r0 + g + 8;
#pragma unroll
                for (int n = 0; n < 4; ++n) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int j = sb0 + kb0 + n * 8 + 2 * t + c;
                        if (abs(ia - j) > win.w) sacc[n][c] = -INFINITY;
                        if (abs(ib - j) > win.w) sacc[n][2 + c] = -INFINITY;
                    }
                }
            }
            float bm0 = -INFINITY, bm1 = -INFINITY;
            if (kb0 + 32 > nk) {                     // only the last key block holds keys past the sequence end
#pragma unroll
                for (int n = 0; n < 4; ++n) {
                    const int k0 = kb0 + n * 8 + 2 * t;
                    if (k0 >= nk) { sacc[n][0] = -INFINITY; sacc[n][2] = -INFINITY; }
                    if (k0 + 1 >= nk) { sacc[n][1] = -INFINITY; sacc[n][3] = -INFINITY; }
                }
            }
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                bm0 = fmaxf(bm0, fmaxf(sacc[n][0], sacc[n][1]));
                bm1 = fmaxf(bm1, fmaxf(sacc[n][2], sacc[n][3]));
            }
            bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1));
            bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
            bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1));
            bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
            const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);
            // exponent base: the running max, or 0 while a windowed row has seen masked keys only (see Window)
            const float ms0 = kHasWindow<RelBias...> && mn0 == -INFINITY ? 0.f : mn0;
            const float ms1 = kHasWindow<RelBias...> && mn1 == -INFINITY ? 0.f : mn1;
            const float c0 = fast_exp2(m0 - ms0), c1 = fast_exp2(m1 - ms1);   // scores are pre-scaled by log2(e)
            m0 = mn0; m1 = mn1;
            float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                sacc[n][0] = fast_exp2(sacc[n][0] - ms0); sacc[n][1] = fast_exp2(sacc[n][1] - ms0);
                sacc[n][2] = fast_exp2(sacc[n][2] - ms1); sacc[n][3] = fast_exp2(sacc[n][3] - ms1);
                ps0 += sacc[n][0] + sacc[n][1];
                ps1 += sacc[n][2] + sacc[n][3];
            }
            l0 = l0 * c0 + ps0;
            l1 = l1 * c1 + ps1;
#pragma unroll
            for (int n = 0; n < NT; ++n) { oacc[n][0] *= c0; oacc[n][1] *= c0; oacc[n][2] *= c1; oacc[n][3] *= c1; }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                if (kb0 + kk * 16 < nk16) {
                    uint32_t pfh[4], pfl[4];
                    split_pack(sacc[2 * kk][0], sacc[2 * kk][1], pfh[0], pfl[0]);
                    split_pack(sacc[2 * kk][2], sacc[2 * kk][3], pfh[1], pfl[1]);
                    split_pack(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1], pfh[2], pfl[2]);
                    split_pack(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3], pfh[3], pfl[3]);
                    // ldmatrix.x4.trans: matrices (keys 0-7, d-tile n), (keys 8-15, n), (keys 0-7, n+1), (keys 8-15, n+1)
                    const int krow = kb0 + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                    const int dsel = (lane >> 4) * 8;
                    uint32_t vh4[NT / 2][4], vl4[NT / 2][4];
#pragma unroll
                    for (int n2 = 0; n2 < NT / 2; ++n2) {
                        ldmatrix_x4_trans(vh4[n2], Vh + krow * KSTR + n2 * 16 + dsel);
                        ldmatrix_x4_trans(vl4[n2], Vl + krow * KSTR + n2 * 16 + dsel);
                    }
#pragma unroll
                    for (int n2 = 0; n2 < NT / 2; ++n2) {
                        const uint32_t a_[2] = {vh4[n2][0], vh4[n2][1]}, b_[2] = {vh4[n2][2], vh4[n2][3]};
                        mma16816(oacc[2 * n2], pfh, a_);
                        mma16816(oacc[2 * n2 + 1], pfh, b_);
                    }
#pragma unroll
                    for (int n2 = 0; n2 < NT / 2; ++n2) {
                        const uint32_t a_[2] = {vh4[n2][0], vh4[n2][1]}, b_[2] = {vh4[n2][2], vh4[n2][3]};
                        mma16816(oacc[2 * n2], pfl, a_);
                        mma16816(oacc[2 * n2 + 1], pfl, b_);
                    }
#pragma unroll
                    for (int n2 = 0; n2 < NT / 2; ++n2) {
                        const uint32_t a_[2] = {vl4[n2][0], vl4[n2][1]}, b_[2] = {vl4[n2][2], vl4[n2][3]};
                        mma16816(oacc[2 * n2], pfh, a_);
                        mma16816(oacc[2 * n2 + 1], pfh, b_);
                    }
                }
            }
        }
    }
    if (!warp_live) return;
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const int ra = r0 + g, rb = r0 + g + 8;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        const int col = h * DH + n * 8 + 2 * t;
        uint32_t hi, lo;
        if (ra < qrows) {
            split_pack(oacc[n][0] * i0, oacc[n][1] * i0, hi, lo);
            *reinterpret_cast<uint32_t*>(ctx_hi + static_cast<size_t>(orow + ra) * H + col) = hi;
            *reinterpret_cast<uint32_t*>(ctx_lo + static_cast<size_t>(orow + ra) * H + col) = lo;
        }
        if (rb < qrows) {
            split_pack(oacc[n][2] * i1, oacc[n][3] * i1, hi, lo);
            *reinterpret_cast<uint32_t*>(ctx_hi + static_cast<size_t>(orow + rb) * H + col) = hi;
            *reinterpret_cast<uint32_t*>(ctx_lo + static_cast<size_t>(orow + rb) * H + col) = lo;
        }
    }
}

// sentence-transformers Pooling (mean | cls) + optional Normalize -> out [B, H].  compact (CLS only): the planes hold the
// CLS rows alone, [B, H], and sequence b's is row b instead of row cu[b].
__global__ void __launch_bounds__(256) pool_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo,
                                                   const int* __restrict__ cu, int H, int mode, int normalize, int compact,
                                                   float* __restrict__ out) {
    __shared__ float red[32];
    const int b = blockIdx.x;
    const int t0 = cu[b], S = cu[b + 1] - t0;
    const size_t cls_row = compact ? b : t0;
    float ss = 0.f;
    float vals[4];   // H <= 1024 with 256 threads
    int nv = 0;
    for (int d = threadIdx.x; d < H; d += blockDim.x, ++nv) {
        float v = 0.f;
        if (mode == RMU_POOL_CLS) {
            if (S > 0) v = __half2float(hi[cls_row * H + d]) + __half2float(lo[cls_row * H + d]);
        } else {
            for (int t = 0; t < S; ++t) {
                const size_t o = static_cast<size_t>(t0 + t) * H + d;
                v += __half2float(hi[o]) + __half2float(lo[o]);
            }
            v = v / fmaxf(static_cast<float>(S), 1e-9f);
        }
        vals[nv] = v;
        ss = fmaf(v, v, ss);
    }
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) tot += red[i];
    const float inv = normalize ? 1.0f / fmaxf(sqrtf(tot), 1e-12f) : 1.0f;
    nv = 0;
    for (int d = threadIdx.x; d < H; d += blockDim.x, ++nv) out[static_cast<size_t>(b) * H + d] = vals[nv] * inv;
}

// BertPooler (tanh(W_p h_cls + b_p)) + classifier -> logits [B, num_labels]; head_act RMU_HEAD_GELU: DeBERTa's ContextPooler,
// erf-GELU in place of tanh; RMU_HEAD_RELU: DistilBERT's pre_classifier and ReLU.  An empty sequence has h_cls = 0 (its row
// cu[b] belongs to the next sequence, or lies past T).  compact: h_cls of sequence b is row b of [B, H] planes.
__global__ void __launch_bounds__(256) cls_head_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo,
                                                       const int* __restrict__ cu, int H, int num_labels, int compact,
                                                       const float* __restrict__ pw, const float* __restrict__ pb,
                                                       const float* __restrict__ cw, const float* __restrict__ cb,
                                                       int head_act, float* __restrict__ out) {
    extern __shared__ float sh[];   // h[H], pooled[H]
    float* hcls = sh;
    float* pooled = sh + H;
    const int b = blockIdx.x;
    const int t0 = cu[b], S = cu[b + 1] - t0;
    const size_t o = static_cast<size_t>(compact ? b : t0) * H;
    for (int d = threadIdx.x; d < H; d += blockDim.x) hcls[d] = S > 0 ? __half2float(hi[o + d]) + __half2float(lo[o + d]) : 0.f;
    __syncthreads();
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int j = warp; j < H; j += nw) {
        const float* wr = pw + static_cast<size_t>(j) * H;
        float s = 0.f;
        for (int d = lane_id(); d < H; d += 32) s = fmaf(wr[d], hcls[d], s);
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane_id() == 0) {
            const float x = s + pb[j];
            pooled[j] = head_act == RMU_HEAD_GELU ? gelu_erf(x) : head_act == RMU_HEAD_RELU ? fmaxf(x, 0.f) : tanhf(x);
        }
    }
    __syncthreads();
    for (int c = warp; c < num_labels; c += nw) {
        const float* wr = cw + static_cast<size_t>(c) * H;
        float s = 0.f;
        for (int d = lane_id(); d < H; d += 32) s = fmaf(wr[d], pooled[d], s);
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane_id() == 0) out[static_cast<size_t>(b) * num_labels + c] = s + cb[c];
    }
}

// ModernBERT's head (ModernBertPredictionHead + classifier) on pooled rows p [B, H] fp32 (pool_kernel's CLS or mean, not
// normalised) -> out [B, num_labels] = cw LN(gelu_erf(dw p + db)) + cb, LN with gain ng and shift nb (zeros without
// norm_bias).  One 256-thread block per row; the dense layer's outputs are one warp's fmaf chain each, the LayerNorm's
// mean and variance block reductions in a fixed order.
__global__ void __launch_bounds__(256) mb_head_kernel(const float* __restrict__ pooled, int H, int num_labels,
                                                      const float* __restrict__ dw, const float* __restrict__ db,
                                                      const float* __restrict__ ng, const float* __restrict__ nb, float eps,
                                                      const float* __restrict__ cw, const float* __restrict__ cb,
                                                      float* __restrict__ out) {
    extern __shared__ float sh[];   // p[H], y[H]
    __shared__ float red[32];
    float* pr = sh;
    float* y = sh + H;
    const int b = blockIdx.x;
    for (int d = threadIdx.x; d < H; d += blockDim.x) pr[d] = pooled[static_cast<size_t>(b) * H + d];
    __syncthreads();
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int j = warp; j < H; j += nw) {
        const float* wr = dw + static_cast<size_t>(j) * H;
        float s = 0.f;
        for (int d = lane_id(); d < H; d += 32) s = fmaf(wr[d], pr[d], s);
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane_id() == 0) y[j] = gelu_erf(s + db[j]);
    }
    __syncthreads();
    auto block_sum = [&](float v) {
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane_id() == 0) red[warp] = v;
        __syncthreads();
        float t = 0.f;
        for (int i = 0; i < nw; ++i) t += red[i];
        __syncthreads();
        return t;
    };
    float s = 0.f;
    for (int d = threadIdx.x; d < H; d += blockDim.x) s += y[d];
    const float mean = block_sum(s) / static_cast<float>(H);
    float q = 0.f;
    for (int d = threadIdx.x; d < H; d += blockDim.x) { const float e = y[d] - mean; q = fmaf(e, e, q); }
    const float rstd = 1.0f / sqrtf(block_sum(q) / static_cast<float>(H) + eps);
    for (int d = threadIdx.x; d < H; d += blockDim.x) y[d] = (y[d] - mean) * rstd * ng[d] + nb[d];
    __syncthreads();
    for (int c = warp; c < num_labels; c += nw) {
        const float* wr = cw + static_cast<size_t>(c) * H;
        float t = 0.f;
        for (int d = lane_id(); d < H; d += 32) t = fmaf(wr[d], y[d], t);
        for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
        if (lane_id() == 0) out[static_cast<size_t>(b) * num_labels + c] = t + cb[c];
    }
}

// sentence-transformers Dense on pooled rows: y [B, n_out] = act(W x + b) with x [B, n_in], W [n_out, n_in], b [n_out] or
// null, act RMU_DENSE_IDENTITY or RMU_DENSE_TANH.  A block takes kDenseRows rows and kDenseCols outputs, one warp per
// output at a time, so each W row is read once for kDenseRows rows.  Output j of row r is lane l's fmaf chain over
// d = l, l + 32, ... in order, then a fixed xor tree, then the bias and act: the same operations whatever rows share its
// block, so a row's bits do not depend on the batch it came in.  A plain SIMT kernel: at the ingest shape the projection
// is < 0.01 % of the encoder's FLOPs.  It is a launch of its own rather than part of pool_kernel, whose one block per
// sequence would read all of W once per row.
constexpr int kDenseRows = 8, kDenseCols = 64;
__global__ void __launch_bounds__(256) dense_kernel(const float* __restrict__ x, int B, int n_in, int n_out,
                                                    const float* __restrict__ W, const float* __restrict__ bias, int act,
                                                    float* __restrict__ y) {
    const int r0 = blockIdx.x * kDenseRows;
    const int nr = min(kDenseRows, B - r0);
    const int warp = threadIdx.x >> 5, lane = lane_id();
    const int j_end = min(n_out, static_cast<int>(blockIdx.y + 1) * kDenseCols);
    for (int j = blockIdx.y * kDenseCols + warp; j < j_end; j += blockDim.x >> 5) {
        const float* wr = W + static_cast<size_t>(j) * n_in;
        float s[kDenseRows];
#pragma unroll
        for (int r = 0; r < kDenseRows; ++r) s[r] = 0.f;
        for (int d = lane; d < n_in; d += 32) {
            const float w = __ldg(wr + d);
#pragma unroll
            for (int r = 0; r < kDenseRows; ++r)
                if (r < nr) s[r] = fmaf(w, x[static_cast<size_t>(r0 + r) * n_in + d], s[r]);
        }
#pragma unroll
        for (int r = 0; r < kDenseRows; ++r) {
            float v = s[r];
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (bias) v += bias[j];
            if (act == RMU_DENSE_TANH) v = tanhf(v);
            if (lane == 0 && r < nr) y[static_cast<size_t>(r0 + r) * n_out + j] = v;
        }
    }
}

// sentence-transformers Normalize: y[r] /= max(||y[r]||, 1e-12), one warp per row (lane-strided fmaf chain, xor tree)
__global__ void __launch_bounds__(256) l2_normalize_rows_kernel(float* __restrict__ y, int B, int n) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= B) return;
    float* yr = y + static_cast<size_t>(row) * n;
    float ss = 0.f;
    for (int d = lane_id(); d < n; d += 32) ss = fmaf(yr[d], yr[d], ss);
    for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    for (int d = lane_id(); d < n; d += 32) yr[d] *= inv;
}

// pos[t] = t - cu[b] for token t of sequence b: each row's position within its sequence (the rotary epilogue's input)
__global__ void seq_positions_kernel(const int* __restrict__ cu, int B, int T, int* __restrict__ pos) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    int lo_b = 0, hi_b = B;
    while (hi_b - lo_b > 1) {
        const int mid = (lo_b + hi_b) >> 1;
        if (cu[mid] <= t) lo_b = mid; else hi_b = mid;
    }
    pos[t] = t - cu[lo_b];
}

// row cu[b] of [T, H] planes -> row b of [B, H] planes, bit for bit (zeros for an empty sequence).  H % 8 == 0.
__global__ void gather_cls_rows_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, const int* __restrict__ cu,
                                       int H, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
    const int b = blockIdx.x;
    const int t0 = cu[b];
    const bool empty = cu[b + 1] == t0;
    const uint4* sh = reinterpret_cast<const uint4*>(hi + static_cast<size_t>(t0) * H);
    const uint4* sl = reinterpret_cast<const uint4*>(lo + static_cast<size_t>(t0) * H);
    uint4* dh = reinterpret_cast<uint4*>(out_hi + static_cast<size_t>(b) * H);
    uint4* dl = reinterpret_cast<uint4*>(out_lo + static_cast<size_t>(b) * H);
    for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
        uint4 vh = make_uint4(0, 0, 0, 0), vl = vh;
        if (!empty) { vh = sh[i]; vl = sl[i]; }
        dh[i] = vh;
        dl[i] = vl;
    }
}

__global__ void join_planes_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ out, size_t n) {
    size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __half2float(hi[i]) + __half2float(lo[i]);
}

// CLS-only attention: one CTA per (sequence, head) holds the whole K / V staging buffer (51 KB at d_h = 32 and 147
// tokens, so four CTAs per SM).  The kernel is bound by that latency-bound copy, not by the one query row: with one warp
// per CTA only four warps per SM would issue it, so four warps stage and warp 0 computes.
constexpr int kClsAttWarps = 4;

// E2 on the QKV planes [T, 3H] (q pre-scaled by log2(e) / sqrt(d_h)) of a ragged batch -> ctx planes [T, H], in
// kAttWarps-warp (160-row) CTAs.
// cls_q_hi / cls_q_lo non-null: query row 0 of each sequence only, q from those compact planes [B, H] -> ctx [B, H]
// (the K / V columns of the QKV planes are read as above; their Q columns are not), in kClsAttWarps-warp CTAs.
// The sequence index is gridDim.y, at most 65 535: a larger batch runs in slices of 65 535 sequences, each launch with
// cu (and in CLS mode the compact Q and context rows) offset by the slice start.  Within a slice the grid and the
// kernel are those of one launch, so the heads of a sequence still run together and every row is computed the same.
// rel_bias non-null: the [heads, kRelSpan] table of build_relative_bias_table is added to every score.
// nkeys non-null ([B] int32, full mode without a bias): sequence b attends to its first min(max(nkeys[b], 1), S_b) rows.
// dis non-null (DeBERTa-v2, d_h = 64, neither a bias nor a key limit): the position terms of launch_position_terms are
// added to every score; in CLS mode its c2p rows are the compact CLS rows, offset here per slice.
// window > 0 (ModernBERT's local layers; full mode, none of the above): key j is visible to query i iff
// |i - j| <= window (the Window pack).
constexpr int kMaxGridY = 65535;
static int launch_attention(const __half* qkv_hi, const __half* qkv_lo, const __half* cls_q_hi, const __half* cls_q_lo,
                            const int* cu, int B, int H, int heads, int max_seqlen, __half* ctx_hi, __half* ctx_lo,
                            cudaStream_t st, const float* rel_bias = nullptr, const int* nkeys = nullptr,
                            const Disentangled* dis = nullptr, int window = 0) {
    const int DH = H / heads;
    const bool cls = cls_q_hi != nullptr;
    const bool bias = rel_bias != nullptr;
    const int warps = cls ? kClsAttWarps : kAttWarps;
    if (nkeys && (cls || bias)) {
        set_error("attention: a key limit runs on every query row and without a relative bias");
        return RMU_ERR_ARG;
    }
    if (dis && (bias || nkeys || DH != 64)) {
        set_error("attention: the disentangled position terms run with head_dim 64, without a bias or key limit");
        return RMU_ERR_ARG;
    }
    if (window < 0 || (window > 0 && (cls || bias || nkeys || dis))) {
        set_error("attention: a sliding window (window > 0) runs in full mode, without a bias, key limit or position "
                  "terms");
        return RMU_ERR_ARG;
    }
    ProfScope _ps(PROF_ATTN, st);
    const unsigned zblocks = cls ? 1u : static_cast<unsigned>((max_seqlen + warps * 16 - 1) / (warps * 16));
    // keys resident per CTA: the whole (longest) sequence when it fits, else super-blocks of kKeySB
    const int ksb = std::min(kKeySB, (max_seqlen + 31) / 32 * 32);
    const size_t tab = bias ? kRelSpan * sizeof(float) : 0;
    const size_t smem_max = 4 * sizeof(__half) * static_cast<size_t>(kKeySB) * (DH + 8) + tab;
    const size_t smem = 4 * sizeof(__half) * static_cast<size_t>(ksb) * (DH + 8) + tab;
    auto kern = cls ? (DH == 32 ? attention_planes_kernel<32, 4, kClsAttWarps, true> : attention_planes_kernel<64, 2, kClsAttWarps, true>)
              : DH == 32 ? attention_planes_kernel<32, 2> : attention_planes_kernel<64, 1>;   // d_h = 64 needs > 96 registers
    using Tab = const float*;
    auto bkern = cls ? (DH == 32 ? attention_planes_kernel<32, 4, kClsAttWarps, true, Tab>
                                 : attention_planes_kernel<64, 2, kClsAttWarps, true, Tab>)
                     : (DH == 32 ? attention_planes_kernel<32, 2, kAttWarps, false, Tab>
                                 : attention_planes_kernel<64, 1, kAttWarps, false, Tab>);
    auto lkern = DH == 32 ? attention_planes_kernel<32, 2, kAttWarps, false, KeyLimit>
                          : attention_planes_kernel<64, 1, kAttWarps, false, KeyLimit>;
    auto dkern = cls ? attention_planes_kernel<64, 2, kClsAttWarps, true, Disentangled>
                     : attention_planes_kernel<64, 1, kAttWarps, false, Disentangled>;
    auto wkern = DH == 32 ? attention_planes_kernel<32, 2, kAttWarps, false, Window>
                          : attention_planes_kernel<64, 1, kAttWarps, false, Window>;
    if (window > 0) RMU_CUDA(cudaFuncSetAttribute(wkern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)));
    else if (dis) RMU_CUDA(cudaFuncSetAttribute(dkern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)));
    else if (bias) RMU_CUDA(cudaFuncSetAttribute(bkern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)));
    else if (nkeys) RMU_CUDA(cudaFuncSetAttribute(lkern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)));
    else RMU_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)));
    for (int s0 = 0; s0 < B; s0 += kMaxGridY) {
        const int nb = std::min(kMaxGridY, B - s0);
        // full mode addresses Q and the context by token (cu[b] is absolute), CLS mode by sequence
        const size_t roff = cls ? static_cast<size_t>(s0) * H : 0;
        dim3 pg(static_cast<unsigned>(heads), static_cast<unsigned>(nb), zblocks);
        if (window > 0) {
            wkern<<<pg, warps * 32, smem, st>>>(qkv_hi, qkv_lo, nullptr, nullptr, cu + s0, H, ksb, ctx_hi, ctx_lo, Window{window});
        } else if (dis) {
            Disentangled d = *dis;
            if (cls) d.c2p += static_cast<size_t>(s0) * heads * d.W;
            dkern<<<pg, warps * 32, smem, st>>>(qkv_hi, qkv_lo, cls ? cls_q_hi + roff : nullptr, cls ? cls_q_lo + roff : nullptr,
                                                cu + s0, H, ksb, ctx_hi + roff, ctx_lo + roff, d);
        } else if (nkeys)
            lkern<<<pg, warps * 32, smem, st>>>(qkv_hi, qkv_lo, nullptr, nullptr, cu + s0, H, ksb, ctx_hi, ctx_lo,
                                                KeyLimit{nkeys + s0});
        else if (bias)
            bkern<<<pg, warps * 32, smem, st>>>(qkv_hi, qkv_lo, cls ? cls_q_hi + roff : nullptr, cls ? cls_q_lo + roff : nullptr,
                                                cu + s0, H, ksb, ctx_hi + roff, ctx_lo + roff, rel_bias);
        else
            kern<<<pg, warps * 32, smem, st>>>(qkv_hi, qkv_lo, cls ? cls_q_hi + roff : nullptr, cls ? cls_q_lo + roff : nullptr,
                                               cu + s0, H, ksb, ctx_hi + roff, ctx_lo + roff);
        count_launch();
        RMU_CHECK_LAUNCH();
    }
    return RMU_OK;
}

// E3 ln_kernel: LayerNorm of T fp32 rows of H -> split planes.  8 warps (tokens) per block.
static int launch_layernorm(const float* pre, int T, int H, const float* g, const float* b, float eps, __half* hi,
                            __half* lo, cudaStream_t st) {
    constexpr int wpb = 8;
    ProfScope _ps(PROF_LN, st);
    ln_kernel<<<static_cast<unsigned>((T + wpb - 1) / wpb), wpb * 32, 0, st>>>(pre, T, H, g, b, eps, hi, lo);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// E3 embed_ln_kernel: word + token-type + position rows of T tokens of a ragged batch -> LayerNorm -> planes [T, H].
// 8 warps (tokens) per block.  pos_mode: RMU_POS_ABSOLUTE or RMU_POS_OFFSET.
static int launch_embed_ln(const int* ids, const int* type_ids, const int* cu, int B, int T, int H, int vocab, int max_pos,
                           int type_vocab, const float* word, const float* pos, const float* typ, const float* g,
                           const float* b, float eps, __half* hi, __half* lo, cudaStream_t st, int pos_mode = RMU_POS_ABSOLUTE) {
    constexpr int wpb = 8;
    ProfScope _ps(PROF_EMBED, st);
    auto kern = pos_mode == RMU_POS_OFFSET ? embed_ln_kernel<RMU_POS_OFFSET> : embed_ln_kernel<RMU_POS_ABSOLUTE>;
    kern<<<static_cast<unsigned>((T + wpb - 1) / wpb), wpb * 32, 0, st>>>(ids, type_ids, cu, B, T, H, vocab, max_pos,
                                                                          type_vocab, word, pos, typ, g, b, eps, hi, lo);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// E4 pool_kernel: one 256-thread block per sequence -> out [B, H] (H <= 1024: four columns per thread)
static int launch_pool(const __half* hi, const __half* lo, const int* cu, int B, int H, int mode, int normalize, bool compact,
                       float* out, cudaStream_t st) {
    ProfScope _ps(PROF_POOL_HEAD, st);
    pool_kernel<<<B, 256, 0, st>>>(hi, lo, cu, H, mode, normalize, compact ? 1 : 0, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// E4 cls_head_kernel: one 256-thread block per sequence, h_cls and the pooled vector in shared memory -> out [B, num_labels]
static int launch_cls_head(const __half* hi, const __half* lo, const int* cu, int B, int H, int num_labels, bool compact,
                           const float* pw, const float* pb, const float* cw, const float* cb, float* out, cudaStream_t st,
                           int head_act = RMU_HEAD_TANH) {
    ProfScope _ps(PROF_POOL_HEAD, st);
    cls_head_kernel<<<B, 256, 2 * H * sizeof(float), st>>>(hi, lo, cu, H, num_labels, compact ? 1 : 0, pw, pb, cw, cb,
                                                           head_act, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// E4 dense_kernel, then l2_normalize_rows_kernel when normalize: x [B, n_in] -> y [B, n_out]
static int launch_dense(const float* x, int B, int n_in, int n_out, const float* W, const float* b, int act, int normalize,
                        float* y, cudaStream_t st) {
    ProfScope _ps(PROF_POOL_HEAD, st);
    dense_kernel<<<dim3((B + kDenseRows - 1) / kDenseRows, (n_out + kDenseCols - 1) / kDenseCols), 256, 0, st>>>(
        x, B, n_in, n_out, W, b, act, y);
    count_launch();
    RMU_CHECK_LAUNCH();
    if (normalize) {
        l2_normalize_rows_kernel<<<(B + 7) / 8, 256, 0, st>>>(y, B, n_out);
        count_launch();
        RMU_CHECK_LAUNCH();
    }
    return RMU_OK;
}

// E4 mb_head_kernel: one 256-thread block per pooled row -> out [B, num_labels]
static int launch_mb_head(const float* pooled, int B, int H, int num_labels, const float* dw, const float* db,
                          const float* ng, const float* nb, float eps, const float* cw, const float* cb, float* out,
                          cudaStream_t st) {
    ProfScope _ps(PROF_POOL_HEAD, st);
    mb_head_kernel<<<B, 256, 2 * H * sizeof(float), st>>>(pooled, H, num_labels, dw, db, ng, nb, eps, cw, cb, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

static int launch_seq_positions(const int* cu, int B, int T, int* pos, cudaStream_t st) {
    ProfScope _ps(PROF_MISC, st);
    seq_positions_kernel<<<static_cast<unsigned>((T + 255) / 256), 256, 0, st>>>(cu, B, T, pos);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// row cu[b] of the hidden-state planes [T, H] -> compact planes [B, H]: one 128-thread block per sequence
static int launch_gather_cls_rows(const __half* hi, const __half* lo, const int* cu, int B, int H, __half* out_hi,
                                  __half* out_lo, cudaStream_t st) {
    ProfScope _ps(PROF_MISC, st);
    gather_cls_rows_kernel<<<B, 128, 0, st>>>(hi, lo, cu, H, out_hi, out_lo);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// n fp32 values -> (hi, lo) planes; n = 0 launches nothing
static int launch_split_planes(const float* src, size_t n, __half* hi, __half* lo, cudaStream_t st) {
    if (n == 0) return RMU_OK;
    split_planes_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(src, hi, lo, n);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// hi + lo -> n fp32 values; n = 0 launches nothing
static int launch_join_planes(const __half* hi, const __half* lo, size_t n, float* out, cudaStream_t st) {
    if (n == 0) return RMU_OK;
    join_planes_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(hi, lo, out, n);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// MPNet's relative_position_bucket (transformers MPNetEncoder, num_buckets 32, max_distance 128) of rel = key - query:
// keys after the query take buckets 16..31, keys before it 0..15; distances below 8 are exact, larger ones log-spaced
// (the float32 log and the truncation of torch's version) and saturate at bucket 15 from distance 91 on.
static int relative_bucket(int rel) {
    constexpr int kHalf = 16, kExact = 8;
    const int n = rel < 0 ? -rel : rel;
    const int base = rel > 0 ? kHalf : 0;
    if (n < kExact) return base + n;
    const int large = kExact + static_cast<int>(logf(static_cast<float>(n) / kExact) / logf(16.0f) * (kHalf - kExact));
    return base + std::min(large, kHalf - 1);
}

// bias [32, heads] (the checkpoint's relative_attention_bias.weight) -> out [heads, kRelSpan]: entry (h, r + kRelMax) is
// bias[bucket(r), h] * log2(e) for r = key - query in [-kRelMax, kRelMax], in the log2 units of the attention scores
static void build_relative_bias_table(const float* bias, int heads, float* out) {
    for (int h = 0; h < heads; ++h)
        for (int r = -kRelMax; r <= kRelMax; ++r)
            out[static_cast<size_t>(h) * kRelSpan + r + kRelMax] = bias[relative_bucket(r) * heads + h] * 1.4426950408889634f;
}

// ---------------------------------------------------------------------------------------------------- DeBERTa-v2
// transformers' make_log_bucket_position(r, s, max_position) in its float32 arithmetic: r itself for |r| <= s / 2, else
// sign(r) (ceil(log(|r| / mid) / log((max_position - 1) / mid) (mid - 1)) + mid).  Built on the host only: a ceil
// boundary can flip with a device logf.
static int log_bucket(int r, int s, int max_position) {
    const int mid = s / 2;
    const int a = r < 0 ? -r : r;
    if (a <= mid) return r;
    const float lp = ceilf(logf(static_cast<float>(a) / static_cast<float>(mid)) /
                           logf(static_cast<float>(static_cast<double>(max_position - 1) / mid)) * static_cast<float>(mid - 1)) +
                     static_cast<float>(mid);
    return r < 0 ? -static_cast<int>(lp) : static_cast<int>(lp);
}

// the row of the relative embeddings query i uses for key j: cidx[r + rmax] = clamp(s + bucket(r), 0, 2s - 1), r = i - j
// in [-rmax, rmax].  It is non-decreasing in r (bucket is).
static void build_position_index(int s, int max_position, int rmax, int* cidx) {
    for (int r = -rmax; r <= rmax; ++r) cidx[r + rmax] = std::min(std::max(s + log_bucket(r, s, max_position), 0), 2 * s - 1);
}

// P1 position_terms_kernel: out[r, h, w] = a_r,h . p_(c0 + w),h over the head's DH columns, fp32 (hi + lo of both operands
// joined), for r < rows and w < W.  a: split planes with row pitch a_ld (the Q or K columns of the QKV planes, or the
// compact CLS Q planes); p: the PQ' | PK planes [2s, 2H], pitch p_ld, starting at the wanted half.  A CTA computes 32
// rows x 64 relative positions of one head; a thread two rows x four positions, each an fmaf chain over d in order.
constexpr int kPosRows = 32, kPosCols = 64;
template <int DH>
__global__ void __launch_bounds__(256) position_terms_kernel(const __half* __restrict__ a_hi, const __half* __restrict__ a_lo,
                                                             size_t a_ld, int rows, const __half* __restrict__ p_hi,
                                                             const __half* __restrict__ p_lo, size_t p_ld, int c0, int W,
                                                             float* __restrict__ out) {
    __shared__ float As[kPosRows][DH + 1];
    __shared__ float Ps[kPosCols][DH + 1];
    const int h = blockIdx.z, heads = gridDim.z;
    const int r0 = blockIdx.y * kPosRows, w0 = blockIdx.x * kPosCols;
    for (int e = threadIdx.x; e < kPosRows * DH; e += blockDim.x) {
        const int r = e / DH, d = e % DH;
        float v = 0.f;
        if (r0 + r < rows) {
            const size_t o = static_cast<size_t>(r0 + r) * a_ld + h * DH + d;
            v = __half2float(a_hi[o]) + __half2float(a_lo[o]);
        }
        As[r][d] = v;
    }
    for (int e = threadIdx.x; e < kPosCols * DH; e += blockDim.x) {
        const int w = e / DH, d = e % DH;
        float v = 0.f;
        if (w0 + w < W) {
            const size_t o = static_cast<size_t>(c0 + w0 + w) * p_ld + h * DH + d;
            v = __half2float(p_hi[o]) + __half2float(p_lo[o]);
        }
        Ps[w][d] = v;
    }
    __syncthreads();
    const int tr = threadIdx.x >> 4, tc = threadIdx.x & 15;     // rows tr, tr + 16; positions tc + 16 k
    float acc[2][4] = {};
#pragma unroll 8
    for (int d = 0; d < DH; ++d) {
        const float x0 = As[tr][d], x1 = As[tr + 16][d];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float p = Ps[tc + 16 * k][d];
            acc[0][k] = fmaf(x0, p, acc[0][k]);
            acc[1][k] = fmaf(x1, p, acc[1][k]);
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = r0 + tr + 16 * i;
        if (r >= rows) continue;
        float* o = out + (static_cast<size_t>(r) * heads + h) * W + w0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (w0 + tc + 16 * k < W) o[tc + 16 * k] = acc[i][k];
    }
}

// P1 on `rows` rows of a (row pitch a_ld) against the p half (PK for C2P, PQ' for P2C) -> out [rows, heads, W].
// rows = 0 launches nothing.
static int launch_position_terms(const __half* a_hi, const __half* a_lo, size_t a_ld, int rows, const __half* p_hi,
                                 const __half* p_lo, size_t p_ld, int heads, int DH, int c0, int W, float* out,
                                 cudaStream_t st) {
    if (rows == 0) return RMU_OK;
    if (DH != 64 || (rows + kPosRows - 1) / kPosRows > kMaxGridY) {
        set_error("position terms: head_dim must be 64 and a call at most 65535 * 32 rows");
        return RMU_ERR_ARG;
    }
    ProfScope _ps(PROF_ATTN, st);
    dim3 grid(static_cast<unsigned>((W + kPosCols - 1) / kPosCols), static_cast<unsigned>((rows + kPosRows - 1) / kPosRows),
              static_cast<unsigned>(heads));
    position_terms_kernel<64><<<grid, 256, 0, st>>>(a_hi, a_lo, a_ld, rows, p_hi, p_lo, p_ld, c0, W, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// The relative positions a call with sequences of at most max_seqlen tokens reaches: c0 and W of cidx over
// |r| <= max_seqlen - 1 (cidx spans [-rmax, rmax], rmax >= max_seqlen - 1).
static void position_window(const int* cidx_h, int rmax, int max_seqlen, int* c0, int* W) {
    const int m = std::max(std::min(max_seqlen - 1, rmax), 0);
    *c0 = cidx_h[rmax - m];
    *W = cidx_h[rmax + m] - *c0 + 1;
}

// E2 with DeBERTa's position terms on caller-owned planes: P1 twice into ws (C2P of the query rows, P2C of every key),
// then E2 with the Disentangled pack.  pos planes [2s, 2H] = PQ' | PK; cidx_d (device) / cidx_h (host) from
// build_position_index with rmax.  cls_q non-null: the compact Q planes [B, H] of the CLS rows.  ws holds
// (qrows + T) heads W floats, qrows = B (CLS) or T.
static int run_disentangled_attention(const __half* qkv_hi, const __half* qkv_lo, const __half* cls_q_hi,
                                      const __half* cls_q_lo, const int* cu, int B, int T, int H, int heads, int max_seqlen,
                                      const __half* pos_hi, const __half* pos_lo, const int* cidx_d, const int* cidx_h,
                                      int rmax, float* ws, __half* ctx_hi, __half* ctx_lo, cudaStream_t st) {
    const int DH = H / heads;
    const bool cls = cls_q_hi != nullptr;
    int c0 = 0, W = 0;
    position_window(cidx_h, rmax, max_seqlen, &c0, &W);
    const int qrows = cls ? B : T;
    float* c2p = ws;
    float* p2c = ws + static_cast<size_t>(qrows) * heads * W;
    const size_t ld3 = static_cast<size_t>(3) * H, p_ld = static_cast<size_t>(2) * H;
    int rc = cls ? launch_position_terms(cls_q_hi, cls_q_lo, H, B, pos_hi + H, pos_lo + H, p_ld, heads, DH, c0, W, c2p, st)
                 : launch_position_terms(qkv_hi, qkv_lo, ld3, T, pos_hi + H, pos_lo + H, p_ld, heads, DH, c0, W, c2p, st);
    if (rc != RMU_OK) return rc;
    rc = launch_position_terms(qkv_hi + H, qkv_lo + H, ld3, T, pos_hi, pos_lo, p_ld, heads, DH, c0, W, p2c, st);
    if (rc != RMU_OK) return rc;
    const Disentangled dis{c2p, p2c, cidx_d, rmax, c0, W};
    return launch_attention(qkv_hi, qkv_lo, cls_q_hi, cls_q_lo, cu, B, H, heads, max_seqlen, ctx_hi, ctx_lo, st, nullptr,
                            nullptr, &dis);
}

// floats of run_disentangled_attention's workspace
static size_t position_ws_floats(const int* cidx_h, int rmax, int max_seqlen, int qrows, int T, int heads) {
    int c0 = 0, W = 0;
    position_window(cidx_h, rmax, max_seqlen, &c0, &W);
    return (static_cast<size_t>(qrows) + T) * heads * W;
}

// ---------------------------------------------------------------------------------------------------- ColBERT
// C1 colbert_normalize_kernel: fp32 projections proj [T, ld] (ColBERT's `linear`, columns dim..ld zero padding) -> unit
// token vectors out [T, dim] = x / max(||x||, 1e-12) (F.normalize).  keep [T] (null = all kept): a dropped token (the
// punctuation skiplist) is written as zeros; MaxSim skips it by the same mask.  One warp per token.
__global__ void colbert_normalize_kernel(const float* __restrict__ proj, int T, int ld, int dim, const uint8_t* __restrict__ keep,
                                         float* __restrict__ out) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= T) return;
    const int lane = static_cast<int>(lane_id());
    const float* row = proj + static_cast<size_t>(t) * ld;
    float ss = 0.f;
    for (int c = lane; c < dim; c += 32) ss = fmaf(row[c], row[c], ss);
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    const bool kept = keep == nullptr || keep[t] != 0;
    float* dst = out + static_cast<size_t>(t) * dim;
    for (int c = lane; c < dim; c += 32) dst[c] = kept ? row[c] / nrm : 0.f;
}

// C2 colbert_maxsim_kernel: one CTA per (query, document) pair -> out[p] = sum over the query's tokens i of
// max over the document's kept tokens j of q_i . d_j.  A dot product is one thread's fmaf chain over the dims in order;
// warp w takes query tokens w, w + kMaxSimWarps, ... and adds their maxima in that order; thread 0 adds the warps' sums
// in warp order.  So a pair's score depends on its two token lists alone, not on the batch or the grid.  A document
// without a kept token has max -inf (callers refuse that case: [CLS], the marker and [SEP] are always kept).
constexpr int kMaxSimWarps = 8;
__global__ void __launch_bounds__(kMaxSimWarps * 32) colbert_maxsim_kernel(
        const float* __restrict__ q, const int* __restrict__ q_cu, const float* __restrict__ d, const int* __restrict__ d_cu,
        const uint8_t* __restrict__ d_keep, int dim, const int* __restrict__ pair_q, const int* __restrict__ pair_d,
        float* __restrict__ out) {
    __shared__ float part[kMaxSimWarps];
    const int p = blockIdx.x;
    const int qi = pair_q[p], di = pair_d[p];
    const int q0 = q_cu[qi], nq = q_cu[qi + 1] - q0, d0 = d_cu[di], nd = d_cu[di + 1] - d0;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc = 0.f;
    for (int i = warp; i < nq; i += kMaxSimWarps) {
        const float* qv = q + static_cast<size_t>(q0 + i) * dim;
        float m = -INFINITY;
        for (int j = lane; j < nd; j += 32) {
            if (d_keep != nullptr && d_keep[d0 + j] == 0) continue;
            const float* dv = d + static_cast<size_t>(d0 + j) * dim;
            float s = 0.f;
            for (int c = 0; c < dim; ++c) s = fmaf(__ldg(qv + c), __ldg(dv + c), s);
            m = fmaxf(m, s);
        }
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        acc += m;
    }
    if (lane == 0) part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kMaxSimWarps; ++w) s += part[w];
        out[p] = s;
    }
}

static int launch_colbert_normalize(const float* proj, int T, int ld, int dim, const uint8_t* keep, float* out, cudaStream_t st) {
    constexpr int wpb = 8;
    ProfScope _ps(PROF_POOL_HEAD, st);
    colbert_normalize_kernel<<<static_cast<unsigned>((T + wpb - 1) / wpb), wpb * 32, 0, st>>>(proj, T, ld, dim, keep, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// n_pairs = 0 launches nothing
static int launch_colbert_maxsim(const float* q, const int* q_cu, const float* d, const int* d_cu, const uint8_t* d_keep,
                                 int dim, const int* pair_q, const int* pair_d, int n_pairs, float* out, cudaStream_t st) {
    if (n_pairs == 0) return RMU_OK;
    ProfScope _ps(PROF_POOL_HEAD, st);
    colbert_maxsim_kernel<<<static_cast<unsigned>(n_pairs), kMaxSimWarps * 32, 0, st>>>(q, q_cu, d, d_cu, d_keep, dim, pair_q,
                                                                                      pair_d, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}


// ------------------------------------------------------------------------------------ Qwen3
// Qwen3 runs as an encoder on an fp32 residual stream.  Its GEMM and attention inputs are split fp16 planes, which
// cannot hold |x| > 65504: every kernel that writes such planes here sets *flag (when non-null) on a value outside that
// range or a NaN, and the forward reports it instead of returning what the overflow made of the output.
constexpr int kQwenHD = 128;                  // head_dim (the only one the kernels take)
constexpr int kRmsThreads = 128;              // rms_split_kernel: thread i holds columns i, i + 128, ... (H <= 4096)
constexpr int kRmsWideThreads = 256;          // its wide form: columns i, i + 256, ... (4096 < H <= 8192)
constexpr int kRmsMaxPerThread = 32;
constexpr int kRmsMaxHidden = kRmsWideThreads * kRmsMaxPerThread;

__device__ __forceinline__ bool outside_f16(float v) { return !(fabsf(v) <= 65504.0f); }

// the pairwise sum of r[0 .. N): ((r0 + r1) + (r2 + r3)) + ... in a fixed order
template <int N>
__device__ __forceinline__ float pair_tree(const float* r) {
    if constexpr (N == 1) return r[0];
    else return pair_tree<N / 2>(r) + pair_tree<N / 2>(r + N / 2);
}

// Qwen3RMSNorm of one fp32 row per block -> split planes: y = w * (x * (1 / sqrt(mean(x^2) + eps))), all fp32.  The sum
// of squares is per thread in column order, then the warps' shuffle trees, then the warp sums' pairwise tree (four
// warps: (r0 + r1) + (r2 + r3)).  kThreads 128 for H <= 4096; 256 for wider rows, where column c < H is guarded so
// that any multiple of 128 up to 8192 fits.
template <int kThreads>
__global__ void __launch_bounds__(kThreads) rms_split_kernel(const float* __restrict__ x, int H, const float* __restrict__ w,
                                                             float eps, __half* __restrict__ hi, __half* __restrict__ lo,
                                                             int* __restrict__ flag) {
    __shared__ float red[kThreads / 32];
    const size_t row = blockIdx.x;
    const float* xr = x + row * H;
    float v[kRmsMaxPerThread];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kRmsMaxPerThread; ++i)
        if (i * kThreads + static_cast<int>(threadIdx.x) < H) {
            v[i] = xr[i * kThreads + threadIdx.x];
            ss = fmaf(v[i], v[i], ss);
        }
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    const float rs = 1.0f / sqrtf(pair_tree<kThreads / 32>(red) / static_cast<float>(H) + eps);
    bool bad = false;
#pragma unroll
    for (int i = 0; i < kRmsMaxPerThread; ++i) {
        const int c = i * kThreads + threadIdx.x;
        if (c < H) {
            const float y = w[c] * (v[i] * rs);
            __half h, l;
            split_f16(y, h, l);
            hi[row * H + c] = h;
            lo[row * H + c] = l;
            bad |= outside_f16(y);
        }
    }
    if (bad && flag) atomicOr(flag, 1);
}

// h = embed_tokens[id] (fp32 rows, ids clamped into [0, vocab)): one float4 per thread
__global__ void embed_rows_kernel(const int* __restrict__ ids, size_t n4, int H, int vocab, const float* __restrict__ table,
                                  float* __restrict__ out) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const size_t t = i / (H / 4), c4 = i % (H / 4);
    int id = ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    reinterpret_cast<float4*>(out)[i] = reinterpret_cast<const float4*>(table + static_cast<size_t>(id) * H)[c4];
}

// Qwen3's q / k step: one warp per (token, head) of the fp32 QKV rows [T, NH 128], NH = heads + 2 kv_heads (the q
// heads, then k, then v); lane l holds dims 4l .. 4l + 3.  q and k heads: RMSNorm over the head with q_norm / k_norm,
// then rotate-half rotary at the token's position, x'[c] = x[c] cos[c] - x[c + 64] sin[c] and x'[c + 64] = x[c + 64]
// cos[c] + x[c] sin[c] for c < 64 (lane l < 16 holds c, lane l + 16 its partner), and q times qscale (log2(e) / sqrt(d),
// the softmax runs in base 2).  Every head leaves as split planes of the same layout.  kQkNorm false (Llama): no
// per-head RMSNorm, qn / kn unread.
template <bool kQkNorm>
__global__ void __launch_bounds__(256) qk_norm_rope_kernel(const float* __restrict__ qkv, int T, int heads, int kv_heads,
                                                           const int* __restrict__ pos, const float* __restrict__ qn,
                                                           const float* __restrict__ kn, float eps, float qscale,
                                                           const float* __restrict__ rcos, const float* __restrict__ rsin,
                                                           int rope_rows, __half* __restrict__ hi, __half* __restrict__ lo,
                                                           int* __restrict__ flag) {
    const int NH = heads + 2 * kv_heads;
    const size_t gw = static_cast<size_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (gw >= static_cast<size_t>(T) * NH) return;
    const int t = static_cast<int>(gw / NH), hh = static_cast<int>(gw % NH);
    const int lane = threadIdx.x & 31;
    const size_t o = gw * kQwenHD + lane * 4;
    const float4 in = *reinterpret_cast<const float4*>(qkv + o);
    float x[4] = {in.x, in.y, in.z, in.w};
    if (hh < heads + kv_heads) {
        if (kQkNorm) {
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) ss = fmaf(x[i], x[i], ss);
            for (int k = 16; k > 0; k >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, k);
            const float rs = 1.0f / sqrtf(ss / static_cast<float>(kQwenHD) + eps);
            const float4 nw = *reinterpret_cast<const float4*>((hh < heads ? qn : kn) + lane * 4);
            x[0] = nw.x * (x[0] * rs); x[1] = nw.y * (x[1] * rs); x[2] = nw.z * (x[2] * rs); x[3] = nw.w * (x[3] * rs);
        }
        int p = pos[t];
        p = p < 0 ? 0 : (p >= rope_rows ? rope_rows - 1 : p);
        const int fi = (lane & 15) * 4;
        const float4 c4 = *reinterpret_cast<const float4*>(rcos + static_cast<size_t>(p) * (kQwenHD / 2) + fi);
        const float4 s4 = *reinterpret_cast<const float4*>(rsin + static_cast<size_t>(p) * (kQwenHD / 2) + fi);
        const float cs[4] = {c4.x, c4.y, c4.z, c4.w}, sn[4] = {s4.x, s4.y, s4.z, s4.w};
        const float sc = hh < heads ? qscale : 1.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float partner = __shfl_xor_sync(0xffffffffu, x[i], 16);
            x[i] = (lane < 16 ? x[i] * cs[i] - partner * sn[i] : x[i] * cs[i] + partner * sn[i]) * sc;
        }
    }
    uint32_t ph[2], pl[2];
    split_pack(x[0], x[1], ph[0], pl[0]);
    split_pack(x[2], x[3], ph[1], pl[1]);
    *reinterpret_cast<uint2*>(hi + o) = make_uint2(ph[0], ph[1]);
    *reinterpret_cast<uint2*>(lo + o) = make_uint2(pl[0], pl[1]);
    const bool bad = outside_f16(x[0]) || outside_f16(x[1]) || outside_f16(x[2]) || outside_f16(x[3]);
    if (bad && flag) atomicOr(flag, 1);
}

// Qwen3's output rows: one 256-thread block per sequence.  The row is the sequence's last (pad_id < 0) or its rightmost
// token whose id != pad_id, the first when there is none (transformers' last_non_pad_token); y = w RMS(x_row) as in
// rms_split_kernel; then out [B, H] = y, L2-normalised when `normalize` (x / max(|x|, 1e-12), sentence-transformers'
// Normalize), or with a head out [B, num_labels] = head . y, one warp's fmaf chain per label.  An empty sequence: zeros.
__global__ void __launch_bounds__(256) last_token_kernel(const float* __restrict__ x, const int* __restrict__ ids,
                                                         const int* __restrict__ cu, int H, const float* __restrict__ w,
                                                         float eps, int pad_id, int normalize, const float* __restrict__ head,
                                                         int num_labels, float* __restrict__ out) {
    extern __shared__ float yrow[];     // [H]
    __shared__ float red[32];
    __shared__ int sel;
    const int b = blockIdx.x;
    const int t0 = cu[b], S = cu[b + 1] - t0;
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5, lane = threadIdx.x & 31;
    const int ow = head ? num_labels : H;
    if (S <= 0) {
        for (int c = threadIdx.x; c < ow; c += blockDim.x) out[static_cast<size_t>(b) * ow + c] = 0.f;
        return;
    }
    if (warp == 0) {
        int r = S - 1;
        if (pad_id >= 0) {
            r = 0;
            for (int k0 = S; k0 > 0; k0 -= 32) {            // windows [k0 - 32, k0), right to left
                const int k = k0 - 32 + lane;
                const unsigned m = __ballot_sync(0xffffffffu, k >= 0 && ids[t0 + k] != pad_id);
                if (m) { r = k0 - 32 + 31 - __clz(static_cast<int>(m)); break; }
            }
        }
        if (lane == 0) sel = r;
    }
    __syncthreads();
    auto block_sum = [&](float v) {
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) red[warp] = v;
        __syncthreads();
        float s = 0.f;
        for (int i = 0; i < nw; ++i) s += red[i];
        __syncthreads();
        return s;
    };
    const float* xr = x + static_cast<size_t>(t0 + sel) * H;
    float ss = 0.f;
    for (int c = threadIdx.x; c < H; c += blockDim.x) { const float v = xr[c]; yrow[c] = v; ss = fmaf(v, v, ss); }
    const float rs = 1.0f / sqrtf(block_sum(ss) / static_cast<float>(H) + eps);
    float s2 = 0.f;
    for (int c = threadIdx.x; c < H; c += blockDim.x) { const float v = w[c] * (yrow[c] * rs); yrow[c] = v; s2 = fmaf(v, v, s2); }
    if (!head) {
        const float tot = block_sum(s2);
        const float inv = normalize ? 1.0f / fmaxf(sqrtf(tot), 1e-12f) : 1.0f;
        for (int c = threadIdx.x; c < H; c += blockDim.x) out[static_cast<size_t>(b) * H + c] = yrow[c] * inv;
        return;
    }
    __syncthreads();
    for (int c = warp; c < num_labels; c += nw) {
        const float* wr = head + static_cast<size_t>(c) * H;
        float s = 0.f;
        for (int d = lane; d < H; d += 32) s = fmaf(wr[d], yrow[d], s);
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) out[static_cast<size_t>(b) * num_labels + c] = s;
    }
}

// ---------------------------------------------------------------------------------------------------
// attention_causal_kernel: Qwen3's causal grouped-query attention at head_dim 128 (mma.sync m16n8k16, fp32 accumulate,
// the three split products hi*hi + lo*hi + hi*lo of the other encoder kernels).  The planes [T, NH 128] hold q (pre-scaled
// by log2(e) / sqrt(128)) | k | v, NH = heads + 2 kv_heads.  One CTA = (sequence, kv head, hpc of the kv head's G =
// heads / kv_heads query heads, a block of 16 rb query rows, rb = 8 / hpc): its K / V are staged once for all hpc query
// heads.  Warp w computes query head w % hpc on rows 16 (w / hpc) .. + 15 of the block.  The keys run in blocks of
// kCausalKB through shared memory with an online softmax, so any length runs; a warp stops at its rows' diagonal and
// masks j > i in the block that crosses it.  Every block a warp reads holds a key <= each of its rows (blocks start at
// multiples of 32, its rows at a multiple of 16), so a row's running max is finite after the first block.  The span
// kernels below compute the same scores: they share the CTA layout (CausalCta), the q fragments (load_q_frags), the
// staging (stage_keys) and the products and mask (score_block) with this kernel.
// ---------------------------------------------------------------------------------------------------
constexpr int kCausalWarps = 8;
constexpr int kCausalKB = 64;                 // keys staged per step
constexpr int kCausalKSTR = kQwenHD + 8;      // staging row pitch in halves: conflict-free ldmatrix rows
constexpr size_t kCausalSmem = 4 * sizeof(__half) * static_cast<size_t>(kCausalKB) * kCausalKSTR;

// The causal CTA layout of attention_causal_kernel and the span kernels, over one sequence of T rows: grid x = kvh *
// (G / hpc) + sub for kv head kvh, grid z = the block of 16 rb query rows from rbase; kend bounds the keys any row of
// the CTA can see.  The warp computes query head qh() on rows r0() .. + 15; it is live when it has a query head and its
// rows start before T.  The warp's coordinates are methods, computed where a kernel uses them (after the span kernels'
// early exit).
struct CausalCta {
    int hpc, T, G, subs, rb, kvh, sub, rbase;
    __device__ __forceinline__ CausalCta(int heads, int kv_heads, int hpc_, int T_)
        : hpc(hpc_), T(T_), G(heads / kv_heads), subs(G / hpc), rb(kCausalWarps / hpc), kvh(blockIdx.x / subs),
          sub(blockIdx.x % subs), rbase(blockIdx.z * 16 * rb) {}
    __device__ __forceinline__ int kend() const { return min(T, rbase + 16 * rb); }
    __device__ __forceinline__ static int warp() { return threadIdx.x >> 5; }
    __device__ __forceinline__ int qh() const { return kvh * G + sub * hpc + warp() % hpc; }
    __device__ __forceinline__ int r0() const { return rbase + 16 * (warp() / hpc); }
    __device__ __forceinline__ bool warp_live() const { return warp() < hpc * rb && r0() < T; }
};

// v reduced over the quad of lanes that share an mma row (lanes 4g .. 4g + 3)
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// the warp's q fragments of rows r0 .. r0 + 15 of head qh (zero past T, and before row `first`) in the sequence whose
// row r is plane row t0 + r - first
__device__ __forceinline__ void load_q_frags(const __half* ph, const __half* pl, size_t ld, int t0, int qh, int r0, int T,
                                             bool live, uint32_t (&qhf)[kQwenHD / 16][4], uint32_t (&qlf)[kQwenHD / 16][4],
                                             int first = 0) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const __half* qhb = ph + static_cast<size_t>(t0) * ld + qh * kQwenHD;
    const __half* qlb = pl + static_cast<size_t>(t0) * ld + qh * kQwenHD;
    const int ra = r0 + g, rc = r0 + g + 8;
    if (first) { qhb -= static_cast<size_t>(first) * ld; qlb -= static_cast<size_t>(first) * ld; }
#pragma unroll
    for (int ks = 0; ks < kQwenHD / 16; ++ks) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { qhf[ks][i] = 0u; qlf[ks][i] = 0u; }
        if (live && ra < T && ra >= first) {
            qhf[ks][0] = *reinterpret_cast<const uint32_t*>(qhb + ra * ld + ks * 16 + 2 * t);
            qlf[ks][0] = *reinterpret_cast<const uint32_t*>(qlb + ra * ld + ks * 16 + 2 * t);
            qhf[ks][2] = *reinterpret_cast<const uint32_t*>(qhb + ra * ld + ks * 16 + 2 * t + 8);
            qlf[ks][2] = *reinterpret_cast<const uint32_t*>(qlb + ra * ld + ks * 16 + 2 * t + 8);
        }
        if (live && rc < T && rc >= first) {
            qhf[ks][1] = *reinterpret_cast<const uint32_t*>(qhb + rc * ld + ks * 16 + 2 * t);
            qlf[ks][1] = *reinterpret_cast<const uint32_t*>(qlb + rc * ld + ks * 16 + 2 * t);
            qhf[ks][3] = *reinterpret_cast<const uint32_t*>(qhb + rc * ld + ks * 16 + 2 * t + 8);
            qlf[ks][3] = *reinterpret_cast<const uint32_t*>(qlb + rc * ld + ks * 16 + 2 * t + 8);
        }
    }
}

// stage keys [sb0, sb0 + kCausalKB) of the sequence whose rows start at row t0, kv column kcol, into Kh / Kl, zeros
// from key `bound` on; kWithV: the values of column vcol go into Vh / Vl in the same loop.  Key k >= split is read
// from row t0 + k + shift (the batched prefill's own cache region after the shared prefix; the defaults fold away).
// The caller synchronises around it.
template <bool kWithV = false>
__device__ __forceinline__ void stage_keys(const __half* ph, const __half* pl, size_t ld, int t0, size_t kcol, int sb0,
                                           int bound, __half* Kh, __half* Kl, size_t vcol = 0, __half* Vh = nullptr,
                                           __half* Vl = nullptr, int split = INT_MAX, int shift = 0) {
    const int nk = min(kCausalKB, bound - sb0);
    for (int e = threadIdx.x; e < kCausalKB * (kQwenHD / 8); e += blockDim.x) {
        const int j = e / (kQwenHD / 8), c8 = (e % (kQwenHD / 8)) * 8;
        uint4 kh = make_uint4(0, 0, 0, 0), kl = kh, vh = kh, vl = kh;
        if (j < nk) {
            const int k = sb0 + j;
            const size_t o = static_cast<size_t>(t0 + k + (k >= split ? shift : 0)) * ld + c8;
            kh = *reinterpret_cast<const uint4*>(ph + o + kcol);
            kl = *reinterpret_cast<const uint4*>(pl + o + kcol);
            if (kWithV) {
                vh = *reinterpret_cast<const uint4*>(ph + o + vcol);
                vl = *reinterpret_cast<const uint4*>(pl + o + vcol);
            }
        }
        *reinterpret_cast<uint4*>(Kh + j * kCausalKSTR + c8) = kh;
        *reinterpret_cast<uint4*>(Kl + j * kCausalKSTR + c8) = kl;
        if (kWithV) {
            *reinterpret_cast<uint4*>(Vh + j * kCausalKSTR + c8) = vh;
            *reinterpret_cast<uint4*>(Vl + j * kCausalKSTR + c8) = vl;
        }
    }
}

// s[n][.] = the warp's 16 x 32 base-2 scores (hi*hi + lo*hi + hi*lo) against the staged keys kb0 .. kb0 + 31, which
// are keys j0 .. j0 + 31 of the sequence; keys j > row are masked to -inf
__device__ __forceinline__ void score_block(const uint32_t (&qhf)[kQwenHD / 16][4], const uint32_t (&qlf)[kQwenHD / 16][4],
                                            const __half* Kh, const __half* Kl, int kb0, int j0, int r0,
                                            float (&sacc)[4][4]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int n = 0; n < 4; ++n) sacc[n][0] = sacc[n][1] = sacc[n][2] = sacc[n][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < kQwenHD / 16; ++ks) {
        uint32_t bh[4][2], bl[4][2];
        const int lrow = (lane & 7) + ((lane >> 4) << 3);
        const int lcol = ks * 16 + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int n2 = 0; n2 < 2; ++n2) {
            uint32_t th[4], tl[4];
            ldmatrix_x4(th, Kh + (kb0 + n2 * 16 + lrow) * kCausalKSTR + lcol);
            ldmatrix_x4(tl, Kl + (kb0 + n2 * 16 + lrow) * kCausalKSTR + lcol);
            bh[2 * n2][0] = th[0]; bh[2 * n2][1] = th[1]; bh[2 * n2 + 1][0] = th[2]; bh[2 * n2 + 1][1] = th[3];
            bl[2 * n2][0] = tl[0]; bl[2 * n2][1] = tl[1]; bl[2 * n2 + 1][0] = tl[2]; bl[2 * n2 + 1][1] = tl[3];
        }
#pragma unroll
        for (int n = 0; n < 4; ++n) mma16816(sacc[n], qhf[ks], bh[n]);
#pragma unroll
        for (int n = 0; n < 4; ++n) mma16816(sacc[n], qlf[ks], bh[n]);
#pragma unroll
        for (int n = 0; n < 4; ++n) mma16816(sacc[n], qhf[ks], bl[n]);
    }
    if (j0 + 31 > r0) {
#pragma unroll
        for (int n = 0; n < 4; ++n) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int j = j0 + n * 8 + 2 * t + c;
                if (j > r0 + g) sacc[n][c] = -INFINITY;
                if (j > r0 + g + 8) sacc[n][2 + c] = -INFINITY;
            }
        }
    }
}

// the block maxima of the thread's rows g (bm0) and g + 8 (bm1) in a score block
__device__ __forceinline__ void block_row_max(const float (&sacc)[4][4], float& bm0, float& bm1) {
    bm0 = -INFINITY;
    bm1 = -INFINITY;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
        bm0 = fmaxf(bm0, fmaxf(sacc[n][0], sacc[n][1]));
        bm1 = fmaxf(bm1, fmaxf(sacc[n][2], sacc[n][3]));
    }
    bm0 = quad_max(bm0);
    bm1 = quad_max(bm1);
}

// The batched prefill (rmu_decoder_generate_batch) runs this kernel on the suffixes of B prompts that share a prefix
// of P tokens (kCached): sequence b is then the P prefix rows and its cu[b + 1] - cu[b] own rows, the planes hold
// only the own rows (row r of the sequence at plane row cu[b] + r - P), and every key comes from the KV cache: key k
// at cache row k when k < P, else k + shift[cu[b]], where the layer's k / v were appended before the launch.  The
// query rows keep their blocks of 16 from the sequence's start, rows before P compute nothing and are not written,
// and the staged keys hold the bits the full launch stages: each row's arithmetic is the full prompt's.  z0 skips the
// row blocks that lie inside the prefix.
struct PrefixKeys {
    const __half* kv = nullptr;           // the layer's cache planes (kv_append_kernel's layout)
    const int* shift = nullptr;           // per plane row: sequence b's own keys start at cache row P + shift[cu[b]]
    int cap = 0, P = 0, z0 = 0;
};

template <bool kCached = false>
__global__ void __launch_bounds__(kCausalWarps * 32, 1) attention_causal_kernel(const __half* __restrict__ ph,
                                                                                 const __half* __restrict__ pl,
                                                                                 const int* __restrict__ cu, int heads,
                                                                                 int kv_heads, int hpc,
                                                                                 __half* __restrict__ ctx_hi,
                                                                                 __half* __restrict__ ctx_lo,
                                                                                 PrefixKeys pk = PrefixKeys{}) {
    constexpr int DH = kQwenHD, KS = DH / 16, NT = DH / 8, KSTR = kCausalKSTR;
    extern __shared__ __align__(16) unsigned char causal_smem[];
    __half* Kh = reinterpret_cast<__half*>(causal_smem);
    __half* Kl = Kh + kCausalKB * KSTR;
    __half* Vh = Kl + kCausalKB * KSTR;
    __half* Vl = Vh + kCausalKB * KSTR;

    const int b = blockIdx.y;
    const int P = kCached ? pk.P : 0;
    const int t0 = cu[b], S = cu[b + 1] - t0 + P;
    CausalCta c(heads, kv_heads, hpc, S);
    if (kCached) c.rbase += pk.z0 * 16 * c.rb;
    if (c.rbase >= S) return;
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const size_t ld = static_cast<size_t>(heads + 2 * kv_heads) * DH;
    const size_t kcol = static_cast<size_t>(heads + c.kvh) * DH, vcol = static_cast<size_t>(heads + kv_heads + c.kvh) * DH;
    const int qh = c.qh(), r0 = c.r0();
    const bool warp_live = c.warp_live() && r0 + 15 >= P;
    // the cache seen as planes of row pitch 128: K hi at kv, K lo at kv + plane, V at 2 planes further
    const size_t plane = static_cast<size_t>(kv_heads) * pk.cap * DH;
    const __half* kph = kCached ? pk.kv : ph;
    const __half* kpl = kCached ? pk.kv + plane : pl;
    const size_t kld = kCached ? static_cast<size_t>(DH) : ld;
    const size_t kkcol = kCached ? static_cast<size_t>(c.kvh) * pk.cap * DH : kcol;
    const size_t kvcol = kCached ? 2 * plane + static_cast<size_t>(c.kvh) * pk.cap * DH : vcol;
    const int kt0 = kCached ? 0 : t0, ksplit = kCached ? P : INT_MAX, kshift = kCached ? pk.shift[t0] : 0;

    uint32_t qhf[KS][4], qlf[KS][4];
    load_q_frags(ph, pl, ld, t0, qh, r0, S, warp_live, qhf, qlf, P);
    float oacc[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) oacc[n][0] = oacc[n][1] = oacc[n][2] = oacc[n][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    const int kend = c.kend();
    for (int sb0 = 0; sb0 < kend; sb0 += kCausalKB) {
        __syncthreads();
        stage_keys<true>(kph, kpl, kld, kt0, kkcol, sb0, kend, Kh, Kl, kvcol, Vh, Vl, ksplit, kshift);
        __syncthreads();
        if (!warp_live) continue;
        for (int kb0 = 0; kb0 < kCausalKB; kb0 += 32) {
            const int j0 = sb0 + kb0;
            if (j0 > r0 + 15) break;                      // above the diagonal of every row of the warp
            float sacc[4][4], bm0, bm1;
            score_block(qhf, qlf, Kh, Kl, kb0, j0, r0, sacc);
            block_row_max(sacc, bm0, bm1);
            const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);
            const float c0 = fast_exp2(m0 - mn0), c1 = fast_exp2(m1 - mn1);
            m0 = mn0; m1 = mn1;
            float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                sacc[n][0] = fast_exp2(sacc[n][0] - mn0); sacc[n][1] = fast_exp2(sacc[n][1] - mn0);
                sacc[n][2] = fast_exp2(sacc[n][2] - mn1); sacc[n][3] = fast_exp2(sacc[n][3] - mn1);
                ps0 += sacc[n][0] + sacc[n][1];
                ps1 += sacc[n][2] + sacc[n][3];
            }
            l0 = l0 * c0 + ps0;
            l1 = l1 * c1 + ps1;
#pragma unroll
            for (int n = 0; n < NT; ++n) { oacc[n][0] *= c0; oacc[n][1] *= c0; oacc[n][2] *= c1; oacc[n][3] *= c1; }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                if (j0 + kk * 16 > r0 + 15) continue;       // every key of the half is masked for every row
                uint32_t pfh[4], pfl[4];
                split_pack(sacc[2 * kk][0], sacc[2 * kk][1], pfh[0], pfl[0]);
                split_pack(sacc[2 * kk][2], sacc[2 * kk][3], pfh[1], pfl[1]);
                split_pack(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1], pfh[2], pfl[2]);
                split_pack(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3], pfh[3], pfl[3]);
                const int krow = kb0 + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                const int dsel = (lane >> 4) * 8;
#pragma unroll
                for (int n2 = 0; n2 < NT / 2; ++n2) {
                    uint32_t vh4[4], vl4[4];
                    ldmatrix_x4_trans(vh4, Vh + krow * KSTR + n2 * 16 + dsel);
                    ldmatrix_x4_trans(vl4, Vl + krow * KSTR + n2 * 16 + dsel);
                    const uint32_t ha[2] = {vh4[0], vh4[1]}, hb[2] = {vh4[2], vh4[3]};
                    const uint32_t la[2] = {vl4[0], vl4[1]}, lb[2] = {vl4[2], vl4[3]};
                    mma16816(oacc[2 * n2], pfh, ha);
                    mma16816(oacc[2 * n2 + 1], pfh, hb);
                    mma16816(oacc[2 * n2], pfl, ha);
                    mma16816(oacc[2 * n2 + 1], pfl, hb);
                    mma16816(oacc[2 * n2], pfh, la);
                    mma16816(oacc[2 * n2 + 1], pfh, lb);
                }
            }
        }
    }
    if (!warp_live) return;
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const int ra = r0 + g, rc = r0 + g + 8;
    const size_t cld = static_cast<size_t>(heads) * DH;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        const int col = qh * DH + n * 8 + 2 * t;
        uint32_t hv, lv;
        if (ra < S && ra >= P) {
            split_pack(oacc[n][0] * i0, oacc[n][1] * i0, hv, lv);
            *reinterpret_cast<uint32_t*>(ctx_hi + static_cast<size_t>(t0 + ra - P) * cld + col) = hv;
            *reinterpret_cast<uint32_t*>(ctx_lo + static_cast<size_t>(t0 + ra - P) * cld + col) = lv;
        }
        if (rc < S && rc >= P) {
            split_pack(oacc[n][2] * i1, oacc[n][3] * i1, hv, lv);
            *reinterpret_cast<uint32_t*>(ctx_hi + static_cast<size_t>(t0 + rc - P) * cld + col) = hv;
            *reinterpret_cast<uint32_t*>(ctx_lo + static_cast<size_t>(t0 + rc - P) * cld + col) = lv;
        }
    }
}

// the causal layout's grid for sequences of up to T rows: hpc query heads per CTA (all of a group of G = heads /
// kv_heads up to 8, else the largest divisor of G up to 8), x = kv_heads * G / hpc CTAs, z = blocks of 16 * (8 / hpc)
// rows
struct CausalGrid {
    int hpc;
    unsigned x, z;
};

static CausalGrid causal_grid(int heads, int kv_heads, int T) {
    const int G = heads / kv_heads;
    int hpc = std::min(G, kCausalWarps);
    while (G % hpc != 0) --hpc;
    const int rows = 16 * (kCausalWarps / hpc);
    return {hpc, static_cast<unsigned>(kv_heads * (G / hpc)), static_cast<unsigned>((T + rows - 1) / rows)};
}

// E3 rms_split_kernel over T rows of H (H % 128 == 0, H <= 8192): the 128-thread form up to 4096, the wide one above
static int launch_rms_split(const float* x, int T, int H, const float* w, float eps, __half* hi, __half* lo, int* flag,
                            cudaStream_t st) {
    if (T <= 0) return RMU_OK;
    ProfScope _ps(PROF_LN, st);
    if (H <= kRmsThreads * kRmsMaxPerThread)
        rms_split_kernel<kRmsThreads><<<static_cast<unsigned>(T), kRmsThreads, 0, st>>>(x, H, w, eps, hi, lo, flag);
    else
        rms_split_kernel<kRmsWideThreads><<<static_cast<unsigned>(T), kRmsWideThreads, 0, st>>>(x, H, w, eps, hi, lo, flag);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

static int launch_embed_rows(const int* ids, int T, int H, int vocab, const float* table, float* out, cudaStream_t st) {
    const size_t n4 = static_cast<size_t>(T) * (H / 4);
    ProfScope _ps(PROF_EMBED, st);
    embed_rows_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, st>>>(ids, n4, H, vocab, table, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// qn == nullptr (Llama): the q / k step without the per-head RMSNorm
static int launch_qk_norm_rope(const float* qkv, int T, int heads, int kv_heads, const int* pos, const float* qn,
                               const float* kn, float eps, float qscale, const float* rcos, const float* rsin, int rope_rows,
                               __half* hi, __half* lo, int* flag, cudaStream_t st) {
    const size_t warps = static_cast<size_t>(T) * (heads + 2 * kv_heads);
    ProfScope _ps(PROF_MISC, st);
    const unsigned grid = static_cast<unsigned>((warps + 7) / 8);
    if (qn)
        qk_norm_rope_kernel<true><<<grid, 256, 0, st>>>(qkv, T, heads, kv_heads, pos, qn, kn, eps, qscale, rcos, rsin,
                                                        rope_rows, hi, lo, flag);
    else
        qk_norm_rope_kernel<false><<<grid, 256, 0, st>>>(qkv, T, heads, kv_heads, pos, qn, kn, eps, qscale, rcos, rsin,
                                                         rope_rows, hi, lo, flag);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

static int launch_last_token(const float* x, const int* ids, const int* cu, int B, int H, const float* w, float eps,
                             int pad_id, int normalize, const float* head, int num_labels, float* out, cudaStream_t st) {
    ProfScope _ps(PROF_POOL_HEAD, st);
    last_token_kernel<<<B, 256, H * sizeof(float), st>>>(x, ids, cu, H, w, eps, pad_id, normalize, head, num_labels, out);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// attention_causal_kernel over a ragged batch; the sequence index is gridDim.y, so batches above 65 535 sequences run
// in slices, each launch with cu offset by the slice start (the token rows stay absolute)
static int launch_attention_causal(const __half* qkv_hi, const __half* qkv_lo, const int* cu, int B, int heads, int kv_heads,
                                   int max_seqlen, __half* ctx_hi, __half* ctx_lo, cudaStream_t st) {
    const CausalGrid cg = causal_grid(heads, kv_heads, max_seqlen);
    ProfScope _ps(PROF_ATTN, st);
    RMU_CUDA(cudaFuncSetAttribute(attention_causal_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kCausalSmem)));
    for (int s0 = 0; s0 < B; s0 += kMaxGridY) {
        const int nb = std::min(kMaxGridY, B - s0);
        const dim3 grid(cg.x, static_cast<unsigned>(nb), cg.z);
        attention_causal_kernel<false><<<grid, kCausalWarps * 32, kCausalSmem, st>>>(qkv_hi, qkv_lo, cu + s0, heads,
                                                                                     kv_heads, cg.hpc, ctx_hi, ctx_lo);
        count_launch();
        RMU_CHECK_LAUNCH();
    }
    return RMU_OK;
}

// the batched prefill's suffix attention (PrefixKeys): B <= kMaxGridY sequences, the longest max_own own rows after
// the prefix
static int launch_attention_cached(const __half* qkv_hi, const __half* qkv_lo, const int* cu, int B, int heads, int kv_heads,
                                   int max_own, PrefixKeys pk, __half* ctx_hi, __half* ctx_lo, cudaStream_t st) {
    const CausalGrid cg = causal_grid(heads, kv_heads, pk.P + max_own);
    pk.z0 = pk.P / (16 * (kCausalWarps / cg.hpc));
    ProfScope _ps(PROF_ATTN, st);
    RMU_CUDA(cudaFuncSetAttribute(attention_causal_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kCausalSmem)));
    const dim3 grid(cg.x, static_cast<unsigned>(B), cg.z - static_cast<unsigned>(pk.z0));
    attention_causal_kernel<true><<<grid, kCausalWarps * 32, kCausalSmem, st>>>(qkv_hi, qkv_lo, cu, heads, kv_heads,
                                                                                cg.hpc, ctx_hi, ctx_lo, pk);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// ---------------------------------------------------------------------------------------------------
// Attention mass over token spans (rmu_decoder_attention_spans): out[a][b] = sum over query heads h, rows i in span a
// and keys j in span b of P_h[i, j], P the causal softmax of one sequence's planes [T, NH 128] as
// attention_causal_kernel reads them, never materialised.  Three kernels:
//   A (spans_rowstat_kernel): per query head and row, the base-2 row max m and sum l = sum_j exp2(s_ij - m) of the
//     causal scores, with attention_causal_kernel's CTA layout (K staged once per kv head for its query heads) and its
//     three-product split mma.sync QK^T; [heads, T] each.
//   B (spans_mass_kernel): the scores again, for 32-key blocks on or below the diagonal that meet a column span of the
//     chunk (kSpanChunk spans per launch, so any span count runs); p = exp2(s - m) / l; each warp adds, per span of the
//     chunk, its masked row sums into its own shared-memory rows [16][kSpanChunk] in key order, then writes
//     M[h][b][i] (fp32) for its rows.  Every span's own keys are summed directly (no prefix differences).
//   C (spans_reduce_kernel): out[a][b] = sum_h sum_{i in a} M[h][b][i] in float64, a fixed thread -> element map and
//     a fixed tree, so the result is deterministic.
// A and B skip every CTA whose rows meet no span.  Spans are [start, end) pairs (device), clamped into [0, T); end <=
// start is empty.
// ---------------------------------------------------------------------------------------------------
constexpr int kSpanChunk = 32;                // column spans per launch of B (one bit each in a warp's mask)
constexpr size_t kSpanKSmem = 2 * sizeof(__half) * static_cast<size_t>(kCausalKB) * kCausalKSTR;

__device__ __forceinline__ void span_bounds(const int* spans, int s, int T, int& lo, int& hi) {
    lo = min(max(spans[2 * s], 0), T);
    hi = min(max(spans[2 * s + 1], lo), T);
}

// 1 when rows [r0, r1) meet some span (block-uniform; every thread of the block calls it)
__device__ __forceinline__ int rows_meet_spans(const int* spans, int n, int T, int r0, int r1) {
    int hit = 0;
    for (int s = threadIdx.x; s < n && !hit; s += blockDim.x) {
        int lo, hi;
        span_bounds(spans, s, T, lo, hi);
        hit = lo < hi && lo < r1 && hi > r0;
    }
    return __syncthreads_or(hit);
}

// A: grid (kv_heads * G / hpc, 1, row blocks of 16 rb rows), kCausalWarps warps; m / l [heads, T]
__global__ void __launch_bounds__(kCausalWarps * 32, 1) spans_rowstat_kernel(const __half* __restrict__ ph,
                                                                              const __half* __restrict__ pl, int T,
                                                                              int heads, int kv_heads, int hpc,
                                                                              const int* __restrict__ spans, int n_spans,
                                                                              float* __restrict__ m_out,
                                                                              float* __restrict__ l_out) {
    extern __shared__ __align__(16) unsigned char span_smem[];
    __half* Kh = reinterpret_cast<__half*>(span_smem);
    __half* Kl = Kh + kCausalKB * kCausalKSTR;
    const CausalCta c(heads, kv_heads, hpc, T);
    if (!rows_meet_spans(spans, n_spans, T, c.rbase, c.kend())) return;
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const size_t ld = static_cast<size_t>(heads + 2 * kv_heads) * kQwenHD;
    const size_t kcol = static_cast<size_t>(heads + c.kvh) * kQwenHD;
    const int qh = c.qh(), r0 = c.r0();
    const bool warp_live = c.warp_live();
    uint32_t qhf[kQwenHD / 16][4], qlf[kQwenHD / 16][4];
    load_q_frags(ph, pl, ld, 0, qh, r0, T, warp_live, qhf, qlf);
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int sb0 = 0; sb0 < c.kend(); sb0 += kCausalKB) {
        __syncthreads();
        stage_keys(ph, pl, ld, 0, kcol, sb0, T, Kh, Kl);
        __syncthreads();
        if (!warp_live) continue;
        for (int kb0 = 0; kb0 < kCausalKB; kb0 += 32) {
            const int j0 = sb0 + kb0;
            if (j0 > r0 + 15) break;
            float sacc[4][4], bm0, bm1;
            score_block(qhf, qlf, Kh, Kl, kb0, j0, r0, sacc);
            block_row_max(sacc, bm0, bm1);
            const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);
            float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                ps0 += fast_exp2(sacc[n][0] - mn0) + fast_exp2(sacc[n][1] - mn0);
                ps1 += fast_exp2(sacc[n][2] - mn1) + fast_exp2(sacc[n][3] - mn1);
            }
            l0 = l0 * fast_exp2(m0 - mn0) + ps0;
            l1 = l1 * fast_exp2(m1 - mn1) + ps1;
            m0 = mn0; m1 = mn1;
        }
    }
    if (!warp_live) return;
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);
    if (t == 0) {
        const size_t o = static_cast<size_t>(qh) * T;
        if (r0 + g < T) { m_out[o + r0 + g] = m0; l_out[o + r0 + g] = l0; }
        if (r0 + g + 8 < T) { m_out[o + r0 + g + 8] = m1; l_out[o + r0 + g + 8] = l1; }
    }
}

// B: grid as A; column spans c0 .. c0 + nc - 1 (nc <= kSpanChunk); M [heads, kSpanChunk, T] fp32, M[h][b][i] = the
// mass row i of head h gives span c0 + b
__global__ void __launch_bounds__(kCausalWarps * 32, 1) spans_mass_kernel(const __half* __restrict__ ph,
                                                                           const __half* __restrict__ pl, int T, int heads,
                                                                           int kv_heads, int hpc,
                                                                           const int* __restrict__ spans, int n_spans,
                                                                           int c0, int nc, const float* __restrict__ m_in,
                                                                           const float* __restrict__ l_in,
                                                                           float* __restrict__ M) {
    extern __shared__ __align__(16) unsigned char span_smem[];
    __half* Kh = reinterpret_cast<__half*>(span_smem);
    __half* Kl = Kh + kCausalKB * kCausalKSTR;
    float* acc = reinterpret_cast<float*>(Kl + kCausalKB * kCausalKSTR);   // [warps][16][kSpanChunk]
    __shared__ int clo[kSpanChunk], chi[kSpanChunk];
    const CausalCta c(heads, kv_heads, hpc, T);
    if (!rows_meet_spans(spans, n_spans, T, c.rbase, c.kend())) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    if (threadIdx.x < kSpanChunk) {
        int lo = 0, hi = 0;
        if (threadIdx.x < nc) span_bounds(spans, c0 + threadIdx.x, T, lo, hi);
        clo[threadIdx.x] = lo;
        chi[threadIdx.x] = hi;
    }
    float* wacc = acc + warp * 16 * kSpanChunk;
    for (int e = lane; e < 16 * kSpanChunk; e += 32) wacc[e] = 0.f;
    __syncthreads();
    // the keys the chunk can see: from its first span start to the CTA's last row
    int kmin = c.kend();
    for (int b = 0; b < nc; ++b)
        if (clo[b] < chi[b]) kmin = min(kmin, clo[b]);
    const size_t ld = static_cast<size_t>(heads + 2 * kv_heads) * kQwenHD;
    const size_t kcol = static_cast<size_t>(heads + c.kvh) * kQwenHD;
    const int qh = c.qh(), r0 = c.r0();
    const bool warp_live = c.warp_live();
    uint32_t qhf[kQwenHD / 16][4], qlf[kQwenHD / 16][4];
    load_q_frags(ph, pl, ld, 0, qh, r0, T, warp_live, qhf, qlf);
    // rows past T take 1 / l = 0, so every p of theirs is 0
    float mr0 = 0.f, mr1 = 0.f, il0 = 0.f, il1 = 0.f;
    if (warp_live && r0 + g < T) { mr0 = m_in[static_cast<size_t>(qh) * T + r0 + g]; il0 = 1.0f / l_in[static_cast<size_t>(qh) * T + r0 + g]; }
    if (warp_live && r0 + g + 8 < T) { mr1 = m_in[static_cast<size_t>(qh) * T + r0 + g + 8]; il1 = 1.0f / l_in[static_cast<size_t>(qh) * T + r0 + g + 8]; }
    for (int sb0 = kmin / kCausalKB * kCausalKB; sb0 < c.kend(); sb0 += kCausalKB) {
        // a staged block that meets no span of the chunk is skipped (block-uniform)
        bool any = false;
        for (int b = 0; b < nc; ++b) any |= clo[b] < chi[b] && clo[b] < sb0 + kCausalKB && chi[b] > sb0;
        if (!any) continue;
        __syncthreads();
        stage_keys(ph, pl, ld, 0, kcol, sb0, T, Kh, Kl);
        __syncthreads();
        if (!warp_live) continue;
        for (int kb0 = 0; kb0 < kCausalKB; kb0 += 32) {
            const int j0 = sb0 + kb0;
            if (j0 > r0 + 15) break;
            const bool meets = lane < nc && clo[lane] < chi[lane] && clo[lane] < j0 + 32 && chi[lane] > j0;
            unsigned mask = __ballot_sync(0xffffffffu, meets);
            if (!mask) continue;
            float sacc[4][4];
            score_block(qhf, qlf, Kh, Kl, kb0, j0, r0, sacc);
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                sacc[n][0] = fast_exp2(sacc[n][0] - mr0) * il0; sacc[n][1] = fast_exp2(sacc[n][1] - mr0) * il0;
                sacc[n][2] = fast_exp2(sacc[n][2] - mr1) * il1; sacc[n][3] = fast_exp2(sacc[n][3] - mr1) * il1;
            }
            while (mask) {
                const int b = __ffs(mask) - 1;
                mask &= mask - 1;
                const int lo = clo[b], hi = chi[b];
                float v0 = 0.f, v1 = 0.f;
#pragma unroll
                for (int n = 0; n < 4; ++n) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int j = j0 + n * 8 + 2 * t + c;
                        if (j >= lo && j < hi) { v0 += sacc[n][c]; v1 += sacc[n][2 + c]; }
                    }
                }
                v0 = quad_sum(v0);
                v1 = quad_sum(v1);
                if (t == 0) {
                    wacc[g * kSpanChunk + b] += v0;
                    wacc[(g + 8) * kSpanChunk + b] += v1;
                }
            }
        }
    }
    if (!warp_live) return;
    __syncwarp();
    for (int e = lane; e < 16 * nc; e += 32) {
        const int b = e / 16, r = e % 16;
        if (r0 + r < T) M[(static_cast<size_t>(qh) * kSpanChunk + b) * T + r0 + r] = wacc[r * kSpanChunk + b];
    }
}

// C: grid (n_spans, nc), 256 threads; out[a * n_spans + c0 + b] = sum_h sum_{i in a} M[h][b][i] in float64
constexpr int kSpanReduceThreads = 256;
__global__ void __launch_bounds__(kSpanReduceThreads) spans_reduce_kernel(const float* __restrict__ M, int T, int heads,
                                                                          const int* __restrict__ spans, int n_spans, int c0,
                                                                          double* __restrict__ out) {
    __shared__ double red[kSpanReduceThreads];
    const int a = blockIdx.x, b = blockIdx.y;
    int lo, hi;
    span_bounds(spans, a, T, lo, hi);
    double s = 0.0;
    for (int h = 0; h < heads; ++h) {
        const float* row = M + (static_cast<size_t>(h) * kSpanChunk + b) * T;
        for (int i = lo + threadIdx.x; i < hi; i += kSpanReduceThreads) s += static_cast<double>(row[i]);
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int k = kSpanReduceThreads / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[static_cast<size_t>(a) * n_spans + c0 + b] = red[0];
}

// workspace floats of launch_attention_spans: m and l [heads, T], M [heads, kSpanChunk, T]
static size_t attention_spans_ws_floats(int T, int heads) {
    return static_cast<size_t>(heads) * T * (2 + kSpanChunk);
}

// A, then per chunk of kSpanChunk column spans B and C -> out [n_spans, n_spans] (device float64)
static int launch_attention_spans(const __half* qkv_hi, const __half* qkv_lo, int T, int heads, int kv_heads,
                                  const int* spans, int n_spans, float* ws, double* out, cudaStream_t st) {
    const CausalGrid cg = causal_grid(heads, kv_heads, T);
    float* m = ws;
    float* l = m + static_cast<size_t>(heads) * T;
    float* M = l + static_cast<size_t>(heads) * T;
    const size_t smem_b = kSpanKSmem + sizeof(float) * kCausalWarps * 16 * kSpanChunk;
    ProfScope _ps(PROF_ATTN, st);
    RMU_CUDA(cudaFuncSetAttribute(spans_rowstat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSpanKSmem)));
    RMU_CUDA(cudaFuncSetAttribute(spans_mass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_b)));
    const dim3 grid(cg.x, 1, cg.z);
    spans_rowstat_kernel<<<grid, kCausalWarps * 32, kSpanKSmem, st>>>(qkv_hi, qkv_lo, T, heads, kv_heads, cg.hpc, spans,
                                                                      n_spans, m, l);
    count_launch();
    RMU_CHECK_LAUNCH();
    for (int c0 = 0; c0 < n_spans; c0 += kSpanChunk) {
        const int nc = std::min(kSpanChunk, n_spans - c0);
        spans_mass_kernel<<<grid, kCausalWarps * 32, smem_b, st>>>(qkv_hi, qkv_lo, T, heads, kv_heads, cg.hpc, spans,
                                                                   n_spans, c0, nc, m, l, M);
        count_launch();
        RMU_CHECK_LAUNCH();
        spans_reduce_kernel<<<dim3(static_cast<unsigned>(n_spans), static_cast<unsigned>(nc)), kSpanReduceThreads, 0, st>>>(
            M, T, heads, spans, n_spans, c0, out);
        count_launch();
        RMU_CHECK_LAUNCH();
    }
    return RMU_OK;
}

#include "rmu_topk.cuh"

// ---------------------------------------------------------------------------------------------------
// Decoding (rmu_decoder_generate).  The KV cache holds, per layer, K and V as split fp16 planes [kv_heads, cap, 128]
// (K hi | K lo | V hi | V lo, each kv_heads cap 128 halves), row p = the token at position p, as the q / k step left
// its rotated k and its v.  kv_append_kernel copies them out of the QKV planes after each layer's q / k step, so the
// prefill's own launches are unchanged.  A decode step's attention is flash-decoding: the keys [0, n) of a kv head are
// cut into splits of kDecChunk keys, one CTA per (kv head, split, group of up to kDecMaxG query heads) computes the
// partial (max, sum, unnormalised output) of each query head, and attention_decode_combine_kernel merges the splits in
// split order.  No atomics: the same inputs give the same bits.
// ---------------------------------------------------------------------------------------------------
constexpr int kDecChunk = 64;                 // keys per split: short serial walks, many CTAs
constexpr int kDecThreads = 128;              // thread d owns output dim d in P.V
constexpr int kDecWarps = kDecThreads / 32;
constexpr int kDecMaxG = 8;                   // query heads per CTA; larger groups take several CTAs (grid z)
constexpr int kDecPart = 2 + kQwenHD;         // a split's partial per query head: m, l, o[128]

// rows [0, T) of the planes [T, NH 128] (q | k | v) -> cache rows pos0 + t of K and V, or with per-row positions
// (the batched decode) rows pos[t] + shift[t]: one uint4 (8 halves) per thread
__global__ void kv_append_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int T, int heads,
                                 int kv_heads, int pos0, int cap, __half* __restrict__ kv, const int* __restrict__ pos,
                                 const int* __restrict__ shift) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const size_t per_tok = static_cast<size_t>(kv_heads) * (kQwenHD / 8);
    if (i >= static_cast<size_t>(T) * per_tok) return;
    const int t = static_cast<int>(i / per_tok), r = static_cast<int>(i % per_tok);
    const int h = r / (kQwenHD / 8), c8 = (r % (kQwenHD / 8)) * 8;
    const size_t ld = static_cast<size_t>(heads + 2 * kv_heads) * kQwenHD;
    const size_t ks = static_cast<size_t>(t) * ld + static_cast<size_t>(heads + h) * kQwenHD + c8;
    const size_t vs = ks + static_cast<size_t>(kv_heads) * kQwenHD;
    const size_t plane = static_cast<size_t>(kv_heads) * cap * kQwenHD;
    const int row = pos ? pos[t] + shift[t] : pos0 + t;
    const size_t d = (static_cast<size_t>(h) * cap + row) * kQwenHD + c8;
    *reinterpret_cast<uint4*>(kv + d) = *reinterpret_cast<const uint4*>(hi + ks);
    *reinterpret_cast<uint4*>(kv + plane + d) = *reinterpret_cast<const uint4*>(lo + ks);
    *reinterpret_cast<uint4*>(kv + 2 * plane + d) = *reinterpret_cast<const uint4*>(hi + vs);
    *reinterpret_cast<uint4*>(kv + 3 * plane + d) = *reinterpret_cast<const uint4*>(lo + vs);
}

// The batched decode's rows (rmu_decoder_generate_batch): grid z = row b * gz + the group block; row b's q sits qld
// halves after row b - 1's, it sees keys [0, pos[b] + 1), key k at cache row k when k < P, else k + shift[b] (the
// shared prefix, then the row's own region), and its partials and context follow the same row order.  The splits still
// count from key 0, so one may straddle P; pos null: one row of n keys at rows 0 .. n - 1.
struct DecRows {
    const int* pos = nullptr;
    const int* shift = nullptr;
    int P = 0, gz = 1;
    size_t qld = 0;
};

// One split of one kv head for query heads g0 .. g0 + ng of its group.  q [heads, 128] planes, pre-scaled by log2(e) /
// sqrt(128) as the q / k step leaves it.  Scores: warp w takes keys w, w + 4, ..., lane l holds dims 4l .. 4l + 3 and
// forms the prefill's three split products qh kh + ql kh + qh kl in one fp32 chain, then a butterfly over the lanes.
// Softmax per query head in base 2: warp g % 4 takes head g, m = max, p = exp2(s - m), l = sum p (lane-strided, then
// a butterfly).  P.V: thread d, keys in order, o += p (vh + vl) (vh + vl is the fp32 value the planes hold).
// part [heads, nsplit, kDecPart] = (m, l, o).
__global__ void __launch_bounds__(kDecThreads) attention_decode_kernel(const __half* __restrict__ qh,
                                                                       const __half* __restrict__ ql,
                                                                       const __half* __restrict__ kv, int heads,
                                                                       int kv_heads, int cap, int n, int nsplit,
                                                                       float* __restrict__ part, DecRows rows) {
    __shared__ float sp[kDecMaxG][kDecChunk];
    __shared__ float sm[kDecMaxG], sl[kDecMaxG];
    const int b = blockIdx.z / rows.gz;
    const int G = heads / kv_heads, kvh = blockIdx.x, split = blockIdx.y, g0 = (blockIdx.z % rows.gz) * kDecMaxG;
    if (rows.pos) n = rows.pos[b] + 1;
    const int ng = min(kDecMaxG, G - g0);
    const int j0 = split * kDecChunk, nk = min(kDecChunk, n - j0);
    if (nk <= 0) return;                          // past this row's keys (a shorter row of the batch)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int P = rows.pos ? rows.P : INT_MAX, sh = rows.pos ? rows.shift[b] : 0;
    const size_t plane = static_cast<size_t>(kv_heads) * cap * kQwenHD;
    // key j0 + j of the split: its cache row's offset from kh
    auto krow = [&](int j) -> size_t {
        const int k = j0 + j;
        return (static_cast<size_t>(kvh) * cap + k + (k >= P ? sh : 0)) * kQwenHD;
    };
    const __half* kh = kv;
    const __half* kl = kh + plane;
    const __half* vh = kh + 2 * plane;
    const __half* vl = kh + 3 * plane;
    qh += b * rows.qld;
    ql += b * rows.qld;
    part += static_cast<size_t>(b) * heads * nsplit * kDecPart;
    float qhr[kDecMaxG][4], qlr[kDecMaxG][4];
#pragma unroll
    for (int g = 0; g < kDecMaxG; ++g) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { qhr[g][i] = 0.f; qlr[g][i] = 0.f; }
        if (g < ng) {
            const size_t o = static_cast<size_t>(kvh * G + g0 + g) * kQwenHD + lane * 4;
            const uint2 h2 = *reinterpret_cast<const uint2*>(qh + o), l2 = *reinterpret_cast<const uint2*>(ql + o);
            const __half2* hp = reinterpret_cast<const __half2*>(&h2);
            const __half2* lp = reinterpret_cast<const __half2*>(&l2);
            const float2 a = __half22float2(hp[0]), b = __half22float2(hp[1]);
            const float2 c = __half22float2(lp[0]), d = __half22float2(lp[1]);
            qhr[g][0] = a.x; qhr[g][1] = a.y; qhr[g][2] = b.x; qhr[g][3] = b.y;
            qlr[g][0] = c.x; qlr[g][1] = c.y; qlr[g][2] = d.x; qlr[g][3] = d.y;
        }
    }
    for (int j = warp; j < nk; j += kDecWarps) {
        const size_t kr = krow(j);
        const uint2 h2 = *reinterpret_cast<const uint2*>(kh + kr + lane * 4);
        const uint2 l2 = *reinterpret_cast<const uint2*>(kl + kr + lane * 4);
        const __half2* hp = reinterpret_cast<const __half2*>(&h2);
        const __half2* lp = reinterpret_cast<const __half2*>(&l2);
        const float2 a = __half22float2(hp[0]), b = __half22float2(hp[1]);
        const float2 c = __half22float2(lp[0]), d = __half22float2(lp[1]);
        const float khf[4] = {a.x, a.y, b.x, b.y}, klf[4] = {c.x, c.y, d.x, d.y};
#pragma unroll
        for (int g = 0; g < kDecMaxG; ++g) {
            if (g >= ng) break;
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                s = fmaf(qhr[g][i], khf[i], s);
                s = fmaf(qlr[g][i], khf[i], s);
                s = fmaf(qhr[g][i], klf[i], s);
            }
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) sp[g][j] = s;
        }
    }
    __syncthreads();
    for (int g = warp; g < ng; g += kDecWarps) {
        float m = -INFINITY;
        for (int j = lane; j < nk; j += 32) m = fmaxf(m, sp[g][j]);
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float l = 0.f;
        for (int j = lane; j < nk; j += 32) { const float p = fast_exp2(sp[g][j] - m); sp[g][j] = p; l += p; }
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        if (lane == 0) { sm[g] = m; sl[g] = l; }
    }
    __syncthreads();
    float acc[kDecMaxG];
#pragma unroll
    for (int g = 0; g < kDecMaxG; ++g) acc[g] = 0.f;
#pragma unroll 8
    for (int j = 0; j < nk; ++j) {
        const size_t kr = krow(j);
        const float v = __half2float(vh[kr + tid]) + __half2float(vl[kr + tid]);
#pragma unroll
        for (int g = 0; g < kDecMaxG; ++g)
            if (g < ng) acc[g] = fmaf(sp[g][j], v, acc[g]);
    }
    for (int g = 0; g < ng; ++g) {
        float* pp = part + (static_cast<size_t>(kvh * G + g0 + g) * nsplit + split) * kDecPart;
        if (tid == 0) { pp[0] = sm[g]; pp[1] = sl[g]; }
        pp[2 + tid] = acc[g];
    }
}

// one block per (row, query head): the row's splits in order, M = max m_s, L = sum l_s exp2(m_s - M), o = sum o_s
// exp2(m_s - M) / L -> the context planes [rows, heads 128]
__global__ void __launch_bounds__(kDecThreads) attention_decode_combine_kernel(const float* __restrict__ part, int nsplit,
                                                                               __half* __restrict__ ctx_hi,
                                                                               __half* __restrict__ ctx_lo,
                                                                               const int* __restrict__ pos, int heads) {
    const int h = blockIdx.x, d = threadIdx.x;
    const int ns = pos ? (pos[h / heads] + kDecChunk) / kDecChunk : nsplit;   // decode_splits(pos + 1)
    const float* p = part + static_cast<size_t>(h) * nsplit * kDecPart;
    float M = -INFINITY;
    for (int s = 0; s < ns; ++s) M = fmaxf(M, p[static_cast<size_t>(s) * kDecPart]);
    float L = 0.f, O = 0.f;
    for (int s = 0; s < ns; ++s) {
        const float* q = p + static_cast<size_t>(s) * kDecPart;
        const float c = fast_exp2(q[0] - M);
        L = fmaf(q[1], c, L);
        O = fmaf(q[2 + d], c, O);
    }
    __half hv, lv;
    split_f16(O / L, hv, lv);
    ctx_hi[static_cast<size_t>(h) * kQwenHD + d] = hv;
    ctx_lo[static_cast<size_t>(h) * kQwenHD + d] = lv;
}

static int decode_splits(int n) { return (n + kDecChunk - 1) / kDecChunk; }

// the partial buffer of launch_attention_decode, in floats
static size_t decode_part_floats(int heads, int n) { return static_cast<size_t>(heads) * decode_splits(n) * kDecPart; }

static int launch_kv_append(const __half* hi, const __half* lo, int T, int heads, int kv_heads, int pos0, int cap,
                            __half* kv, cudaStream_t st, const int* pos = nullptr, const int* shift = nullptr) {
    const size_t n = static_cast<size_t>(T) * kv_heads * (kQwenHD / 8);
    ProfScope _ps(PROF_DECODE_ATTN, st);
    kv_append_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(hi, lo, T, heads, kv_heads, pos0, cap, kv,
                                                                              pos, shift);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// one query row q [heads 128] against cache rows [0, n) of one layer's kv -> ctx [heads 128]; with rows.pos, B rows
// (DecRows) of at most n keys each -> ctx [B, heads 128]
static int launch_attention_decode(const __half* q_hi, const __half* q_lo, const __half* kv, int heads, int kv_heads,
                                   int cap, int n, float* part, __half* ctx_hi, __half* ctx_lo, cudaStream_t st,
                                   int B = 1, DecRows rows = DecRows{}) {
    const int G = heads / kv_heads, ns = decode_splits(n);
    rows.gz = (G + kDecMaxG - 1) / kDecMaxG;
    ProfScope _ps(PROF_DECODE_ATTN, st);
    const dim3 grid(static_cast<unsigned>(kv_heads), static_cast<unsigned>(ns), static_cast<unsigned>(B * rows.gz));
    attention_decode_kernel<<<grid, kDecThreads, 0, st>>>(q_hi, q_lo, kv, heads, kv_heads, cap, n, ns, part, rows);
    count_launch();
    RMU_CHECK_LAUNCH();
    attention_decode_combine_kernel<<<static_cast<unsigned>(B * heads), kDecThreads, 0, st>>>(part, ns, ctx_hi, ctx_lo,
                                                                                               rows.pos, heads);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

__global__ void set_int_kernel(int* p, int v) { *p = v; }

// ---------------------------------------------------------------------------------------------------
// Token selection over fp32 logits [V] (one CTA), in transformers' order:
//   repetition penalty: x = bit(i) ? (x < 0 ? x p : x / p) : x for the ids whose presence bit is set;
//   greedy (do_sample 0): the largest x, the lowest index among equal ones;
//   sampling: x / temperature; top-k keeps every x >= the k-th largest (ties included, but at most kSampleCap
//   candidates: among ties at the k-th value the lowest indices win); top-p over the candidates sorted ascending,
//   dropping those whose cumulative softmax is <= 1 - top_p (the largest always stays); then the inverse CDF: the
//   first candidate, largest first, whose cumulative weight exceeds u times the kept total.
// The candidates are the index's top-k tail (rmu_topk.cuh): keys (score desc, index asc), a radix select of the k-th
// and of the kSampleCap-th key, the keys above the higher of the two, a bitonic sort.  Weights exp(x - max) are float64,
// summed in a fixed order by one thread.  u is u_in when u_in >= 0, else the Philox4x32-10 uniform of (seed, step).
// The chosen id is written to *token and its presence bit set.  The batched decode runs one CTA per live row r
// (SampleRows): logits row r, token r, and the presence bits and Philox seed of the row's sequence seq[r].  A
// prompt-lookup verify pass runs one CTA per row of one sequence: row r has its own presence bits (seq null), the
// call's seed (seeds null) and step + r (row_step), so it samples as the sequential step it stands for.  A decode
// session's rows each carry their own settings and step (args, steps per sequence): row r then samples exactly as
// sequential step steps[seq[r]] of its own request would.
// ---------------------------------------------------------------------------------------------------
constexpr int kSampleThreads = 1024;
constexpr int kSampleCap = 256;               // the largest top_k and the most candidates

struct SampleArgs {
    int do_sample, top_k;
    float temperature, top_p, penalty;
};

struct SampleRows {
    const int* seq = nullptr;                     // row r's sequence; null: r
    const unsigned long long* seeds = nullptr;    // [sequences]; null: `seed` for every row
    size_t words = 0;                             // presence words per sequence; 0: one row, presence at its start
    bool row_step = false;                        // row r draws at step + r
    const SampleArgs* args = nullptr;             // [sequences]; null: `a` for every row
    const unsigned long long* steps = nullptr;    // [sequences]: the sequence's Philox step; null: `step`
};

// Philox4x32-10 (Salmon et al., SC'11) with counter (step, 0) and key seed: the first output word's high 24 bits / 2^24
__host__ __device__ inline float philox_uniform(unsigned long long seed, unsigned long long step) {
    uint32_t c0 = static_cast<uint32_t>(step), c1 = static_cast<uint32_t>(step >> 32), c2 = 0u, c3 = 0u;
    uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
    for (int r = 0; r < 10; ++r) {
        const unsigned long long p0 = 0xD2511F53ull * c0, p1 = 0xCD9E8D57ull * c2;
        const uint32_t hi0 = static_cast<uint32_t>(p0 >> 32), lo0 = static_cast<uint32_t>(p0);
        const uint32_t hi1 = static_cast<uint32_t>(p1 >> 32), lo1 = static_cast<uint32_t>(p1);
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return static_cast<float>(c0 >> 8) * (1.0f / 16777216.0f);
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(float* __restrict__ logits, int V,
                                                                unsigned* __restrict__ presence, SampleArgs a, float u_in,
                                                                unsigned long long seed, unsigned long long step,
                                                                int* __restrict__ token, SampleRows rows) {
    __shared__ unsigned long long sel[kSel2Max];
    __shared__ int hist[256];
    __shared__ unsigned long long s_prefix, s_best[kSampleThreads / 32];
    __shared__ int s_remaining, s_ties, s_cnt;
    __shared__ double w[kSampleCap];
    const int tid = threadIdx.x;
    if (rows.words) {
        const int q = rows.seq ? rows.seq[blockIdx.x] : blockIdx.x;
        logits += static_cast<size_t>(blockIdx.x) * V;
        token += blockIdx.x;
        presence += q * rows.words;
        if (rows.seeds) seed = rows.seeds[q];
        if (rows.row_step) step += blockIdx.x;
        if (rows.args) a = rows.args[q];
        if (rows.steps) step = rows.steps[q];
    }
    unsigned long long best = 0ull;
    for (int i = tid; i < V; i += blockDim.x) {
        float x = logits[i];
        if ((presence[i >> 5] >> (i & 31)) & 1u) x = x < 0.f ? x * a.penalty : __fdiv_rn(x, a.penalty);
        if (a.do_sample) x = __fdiv_rn(x, a.temperature);
        logits[i] = x;
        const unsigned long long k = make_key(x, static_cast<uint32_t>(i));
        best = k > best ? k : best;
    }
    if (!a.do_sample) {
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long b = __shfl_xor_sync(0xffffffffu, best, o); best = b > best ? b : best; }
        if ((tid & 31) == 0) s_best[tid >> 5] = best;
        __syncthreads();
        if (tid == 0) {
            for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) best = s_best[i] > best ? s_best[i] : best;
            const int id = static_cast<int>(key_row(best));
            *token = id;
            presence[id >> 5] |= 1u << (id & 31);
        }
        return;
    }
    __syncthreads();                                            // the tempered logits are visible to the block
    auto load_key = [&](long long i) -> unsigned long long { return make_key(logits[i], static_cast<uint32_t>(i)); };
    const unsigned long long tk = block_radix_select(load_key, V, a.top_k, hist, &s_prefix, &s_remaining, &s_ties);
    __syncthreads();
    const unsigned long long tc = block_radix_select(load_key, V, kSampleCap, hist, &s_prefix, &s_remaining, &s_ties);
    // every key whose score equals the k-th one's is >= (that score, low word 0)
    const unsigned long long tks = tk == 1ull ? 1ull : (tk & 0xFFFFFFFF00000000ull);
    const unsigned long long T = tks > tc ? tks : tc;
    const int n = min(block_collect(load_key, V, T, sel, &s_cnt), kSampleCap);
    block_sort_desc(sel, n);
    const double m = static_cast<double>(key_score(sel[0]));
    for (int r = tid; r < n; r += blockDim.x) w[r] = exp(static_cast<double>(key_score(sel[r])) - m);
    __syncthreads();
    if (tid == 0) {
        double total = 0.0;
        for (int r = 0; r < n; ++r) total += w[r];
        // ascending cumulative softmax of candidate r = the sum over r..n-1; kept: r < nkeep
        int nkeep = n;
        double suf = 0.0;
        for (int r = n - 1; r > 0; --r) {
            suf += w[r];
            if (suf / total <= 1.0 - static_cast<double>(a.top_p)) nkeep = r; else break;
        }
        double kept = 0.0;
        for (int r = 0; r < nkeep; ++r) kept += w[r];
        const double u = u_in >= 0.f ? static_cast<double>(u_in) : static_cast<double>(philox_uniform(seed, step));
        const double target = u * kept;
        int pick = nkeep - 1;
        double cum = 0.0;
        for (int r = 0; r < nkeep; ++r) {
            cum += w[r];
            if (target < cum) { pick = r; break; }
        }
        const int id = static_cast<int>(key_row(sel[pick]));
        *token = id;
        presence[id >> 5] |= 1u << (id & 31);
    }
}

static int launch_sample(float* logits, int V, unsigned* presence, const SampleArgs& a, float u_in, unsigned long long seed,
                         unsigned long long step, int* token, cudaStream_t st, int B = 1, SampleRows rows = SampleRows{}) {
    ProfScope _ps(PROF_SAMPLE, st);
    sample_kernel<<<B, kSampleThreads, 0, st>>>(logits, V, presence, a, u_in, seed, step, token, rows);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

// A verify pass's presence bits: rows [M, words], row j = base | the bits of ids[1 .. j] (the drafts fed before row
// j's own token), one thread per word of a row
__global__ void presence_rows_kernel(const unsigned* __restrict__ base, size_t words, const int* __restrict__ ids, int M,
                                     unsigned* __restrict__ rows) {
    const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= words * M) return;
    const int j = static_cast<int>(i / words);
    const size_t w = i % words;
    unsigned v = base[w];
    for (int d = 1; d <= j; ++d)
        if (static_cast<size_t>(ids[d] >> 5) == w) v |= 1u << (ids[d] & 31);
    rows[i] = v;
}

static int launch_presence_rows(const unsigned* base, size_t words, const int* ids, int M, unsigned* rows, cudaStream_t st) {
    const size_t n = words * M;
    ProfScope _ps(PROF_SAMPLE, st);
    presence_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(base, words, ids, M, rows);
    count_launch();
    RMU_CHECK_LAUNCH();
    return RMU_OK;
}

}  // namespace rmu

using namespace rmu;

struct EncLayer {
    SplitOperand Wqkv, Wo, W1, W2;
    float *bqkv = nullptr, *bo = nullptr, *b1 = nullptr, *b2 = nullptr;
    float *ln1g = nullptr, *ln1b = nullptr, *ln2g = nullptr, *ln2b = nullptr;
    SplitOperand D1, D2;                  // adapter_dim > 0: X-MOD's language adapter, dense1 [A, H] and dense2 [H, A]
    float *d1 = nullptr, *d2 = nullptr;
    __half *pos_hi = nullptr, *pos_lo = nullptr;   // position_buckets > 0: PQ' | PK planes [2s, 2H] of the layer
    int window = 0;                       // ModernBERT: the layer's attention half-window (0 = global attention)
    float *qn = nullptr, *kn = nullptr;   // Qwen3: q_norm, k_norm [128]
    Nf4Weight nf4[4];                     // rmu_decoder_quantize_nf4: Wqkv, Wo, W1, W2 in NF4 (their split planes freed)
};

// A device scratch buffer that only grows.  The caller's lock keeps other users of the buffer out.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;                       // bytes
    template <typename T> T* as() const { return static_cast<T*>(p); }
    void release() { cudaFree(p); p = nullptr; cap = 0; }
};

// make b hold at least `need` bytes; when it must grow it allocates max(need, alloc).  The device is synchronised
// first: work queued on any stream may still read the old allocation.  A failed allocation leaves b empty, clears the
// CUDA error (an out-of-memory is not sticky, so the handle stays usable) and names the bytes it asked for.
static int grow(DevBuf& b, size_t need, size_t alloc = 0) {
    if (need <= b.cap) return RMU_OK;
    RMU_CUDA(cudaDeviceSynchronize());
    b.release();
    alloc = std::max(need, alloc);
    const cudaError_t err = cudaMalloc(&b.p, alloc);
    if (err != cudaSuccess) {
        cudaGetLastError();
        b.p = nullptr;
        set_error("cannot allocate " + std::to_string(alloc) + " bytes of device memory: " + cudaGetErrorString(err));
        return RMU_ERR_CUDA;
    }
    b.cap = alloc;
    return RMU_OK;
}

// Lays regions out back to back at 256-byte boundaries: run a layout once from a null base to size its buffer, then
// again from the buffer to place the regions
struct Carve {
    uintptr_t base;
    size_t size = 0;
    explicit Carve(void* b) : base(reinterpret_cast<uintptr_t>(b)) {}
    template <typename T> T* take(size_t n) {
        T* p = reinterpret_cast<T*>(base + size);
        size += (n * sizeof(T) + 255) / 256 * 256;
        return p;
    }
};

// rows of the per-token and per-sequence buffers grown for T tokens and B sequences
static size_t token_rows(int T) { return (std::max(T, 1024) + 127) / 128 * 128; }
static size_t seq_rows(int B) { return std::max(B + 1, 1024); }

struct rmu_encoder {
    rmu_bert_config cfg{};
    rmu_encoder_ext ext{};                // DeBERTa's fields, zero for every other model
    int has_head = 0, sms = 0, device = 0;
    std::vector<void*> allocs;
    float *word = nullptr, *pos = nullptr, *typ = nullptr, *eg = nullptr, *eb = nullptr;
    float* rel = nullptr;                 // rel_buckets = 32: [heads, kRelSpan] attention bias table, else null
    std::vector<EncLayer> layers;
    SplitOperand last_wq, last_wkv;       // views of the last layer's Wqkv: rows 0..H (q) and H..3H (k | v)
    float *pw = nullptr, *pb = nullptr, *cw = nullptr, *cb = nullptr;
    // ModernBERT (pre-LN, run_modernbert): ln1 = attn_norm (null in layer 0), W1 = Wi with its rows in GeGLU blocks, ln2 =
    // mlp_norm; final_norm; the head's norm (pw / pb = head.dense); rope tables [max_pos, d_h / 2] of global (0) and
    // local (1) layers; the classifier's pooling
    bool modern = false;
    float *fng = nullptr, *fnb = nullptr, *hng = nullptr, *hnb = nullptr;
    float *rope_cos[2] = {nullptr, nullptr}, *rope_sin[2] = {nullptr, nullptr};
    int mb_pool = RMU_POOL_CLS;
    // Qwen3 (run_qwen3): ln1g = input_layernorm, Wqkv = q | k | v proj, Wo = o_proj, ln2g = post_attention_layernorm, W1 =
    // gate | up in 64-row SwiGLU blocks, W2 = down_proj; fng = norm; cw = the last-token head [num_labels, H];
    // rope_cos / rope_sin[0]; zeros = a zero bias for every projection (Qwen3 has none); QKVF the fp32 q | k | v rows
    // before the q / k step; range_flag the fp16-range flag of the split kernels, read back after the layers
    bool qwen = false;
    rmu_qwen3_ext qext{};
    float* zeros = nullptr;
    float* QKVF = nullptr;
    int* range_flag = nullptr;
    // Llama (rmu_encoder_create_llama) runs as Qwen3 with qn = kn = null (no per-head q / k RMSNorm); the span
    // attention's workspace (launch_attention_spans) and its one-sequence cu_seqlens [0, T], grown under mu
    bool llama = false;
    DevBuf span_ws;
    int* span_cu = nullptr;
    // generation (rmu_decoder_set_lm_head, rmu_decoder_generate*): the LM head [V, H] as split planes and a zero bias
    // [V]; the KV cache (layers x K hi | K lo | V hi | V lo [kv_heads, kv_cap, 128]); gen_ws = the scratch of one
    // generate or generate_batch call, laid out by that call.  Grown under mu.
    SplitOperand lm_head;
    bool has_lm_head = false;
    float* lm_zero = nullptr;
    DevBuf kv_cache, gen_ws;
    int kv_cap = 0;
    // NF4 weights (rmu_decoder_quantize_nf4): the layers' projections live in EncLayer::nf4; a prefill dequantises
    // each into the one scratch operand set nf4_hi | nf4_lo (lo all zero), seen through nf4_op[projection]'s tensor
    // maps.  nf4_broken: a conversion failed part-way and the handle cannot run.  nf4_peak / nf4_delta: the most the
    // conversion's allocations exceeded, and finally differ from, the bytes the handle held before it.
    bool nf4 = false, nf4_broken = false;
    __half *nf4_hi = nullptr, *nf4_lo = nullptr;
    // built layer by layer (rmu_decoder_create_nf4): layers 0 .. layers_loaded - 1 hold their weights, and the handle
    // runs nothing until every layer does
    bool by_layer = false;
    int layers_loaded = 0;
    SplitOperand nf4_op[4];
    int64_t nf4_peak = 0, nf4_delta = 0;
    // sentence-transformers Dense modules after pooling (rmu_encoder_set_dense): dense_dims [n + 1], per layer W [out, in],
    // b [out] or null, act; dense_ws holds two [B, max width] ping-pong rows, grown under mu
    std::vector<int> dense_dims;
    std::vector<float*> dense_w, dense_b;
    std::vector<int> dense_act;
    DevBuf dense_ws;
    // activations, in the shape the create path records: QKVP's and CTX's widths, and which optional buffers exist
    // (X1, the CLS rows, QKVF, POSI)
    int tok_cap = 0, seq_cap = 0;
    int qkv_w = 0, ctx_w = 0;
    bool has_x1 = false, has_cls_rows = false, has_qkvf = false, has_posi = false;
    std::vector<void*> act_allocs;
    SplitOperand X, CTX, X1, FF, QKVP;   // QKVP: q (pre-scaled) | k | v as split planes [T, 3H]
    float* PRE = nullptr;                 // fp32 pre-LayerNorm rows: projection + bias + residual
    // the last layer on the CLS rows (run_last_layer_cls): row b = sequence b, [seq_cap, .]; X_cls ends as their hidden state
    SplitOperand X_cls, Q_cls, CTX_cls, X1_cls, FF_cls;
    float* PRE_cls = nullptr;
    SplitOperand FFA, FFA_cls;            // adapter_dim > 0: the FF / FF_cls planes seen as [rows, adapter_dim]
    int* POSI = nullptr;                  // ModernBERT: each token's position within its sequence [tok_cap]
    // position_buckets > 0 (DeBERTa): cidx over |i - j| <= max_pos - 1 (host copy and device table), and the position
    // terms' workspace, grown under mu
    std::vector<int> cidx_h;
    int* cidx = nullptr;
    DevBuf pos_ws;
    // staging of the *_host entry points: owned by host_mu alone (NOT part of the activation workspace, which a
    // concurrent device-pointer caller may free and re-allocate under mu)
    DevBuf d_ids, d_typ, d_cu, d_out;
    cudaEvent_t ws_done = nullptr;   // last use of the shared activation workspace (callers on other streams wait on it)
    std::mutex mu;
    std::mutex host_mu;   // the *_host entry points share the staging buffers above: one at a time per handle
};

// a handle on the current device with cfg and has_head set; null (and `who: no CUDA device`) without a device
static rmu_encoder* new_handle(const std::string& who, const rmu_bert_config& cfg, int has_head) {
    rmu_encoder* e = new rmu_encoder();
    e->cfg = cfg;
    e->has_head = has_head;
    if (cudaGetDevice(&e->device) != cudaSuccess || (e->sms = device_sm_count()) <= 0 ||
        cudaEventCreateWithFlags(&e->ws_done, cudaEventDisableTiming) != cudaSuccess) {
        set_error(who + ": no CUDA device (this library has no CPU path)");
        delete e;
        return nullptr;
    }
    return e;
}

// The GEMM weights travel as split fp16 planes: |w| >= 65520 rounds hi to inf and turns every output it touches into
// NaN.  Refuses the first of the n floats at p outside that range, on the host, before any CUDA call.
static int check_split_range(const std::string& who, const std::string& what, const float* p, size_t n) {
    for (size_t j = 0; j < n; ++j) {
        if (std::fabs(p[j]) >= 65520.0f) {
            set_error(who + ": " + what + " weight [" + std::to_string(j) + "] = " + std::to_string(p[j]) +
                      " is outside the split fp16 planes' range (|w| < 65520)");
            return RMU_ERR_UNSUPPORTED;
        }
    }
    return RMU_OK;
}

template <typename T>
static int dev_alloc(std::vector<void*>& keep, T** p, size_t count) {
    void* q = nullptr;
    RMU_CUDA(cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T)));
    keep.push_back(q);
    *p = static_cast<T*>(q);
    return RMU_OK;
}

static int upload(rmu_encoder* e, float** dst, const float* src_h, size_t n) {
    int rc = dev_alloc(e->allocs, dst, n);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpy(*dst, src_h, n * sizeof(float), cudaMemcpyHostToDevice));
    return RMU_OK;
}

// upload a [rows, cols] fp32 weight (optionally a vertical concat of several) as split fp16 planes
static int upload_split(rmu_encoder* e, SplitOperand* op, const std::vector<const float*>& parts, int rows_each, int cols) {
    const size_t rows = static_cast<size_t>(rows_each) * parts.size();
    const size_t n = rows * cols;
    float* tmp = nullptr;
    RMU_CUDA(cudaMalloc(reinterpret_cast<void**>(&tmp), n * sizeof(float)));
    for (size_t i = 0; i < parts.size(); ++i)
        RMU_CUDA(cudaMemcpy(tmp + i * rows_each * cols, parts[i], static_cast<size_t>(rows_each) * cols * sizeof(float), cudaMemcpyHostToDevice));
    __half *hi = nullptr, *lo = nullptr;
    int rc = dev_alloc(e->allocs, &hi, n);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &lo, n);
    if (rc != RMU_OK) { cudaFree(tmp); return rc; }
    rc = launch_split_planes(tmp, n, hi, lo, nullptr);
    cudaError_t err = cudaDeviceSynchronize();
    cudaFree(tmp);
    if (rc != RMU_OK) return rc;
    if (err != cudaSuccess) { set_error(std::string("split_planes: ") + cudaGetErrorString(err)); return RMU_ERR_CUDA; }
    return make_split_operand(op, hi, lo, static_cast<int64_t>(rows), cols);
}

static void free_acts(rmu_encoder* e) {
    for (void* p : e->act_allocs) cudaFree(p);
    e->act_allocs.clear();
    e->tok_cap = 0;
    e->pos_ws.release();
    e->span_ws.release();
}

// the width rmu_encoder_embed writes: the last Dense module's out_features, else hidden
static int embed_width(const rmu_encoder* e) { return e->dense_dims.empty() ? e->cfg.hidden : e->dense_dims.back(); }

// mu held: the pooled rows (not normalised) -> the Dense chain -> out [B, embed_width], normalised last when asked.
// dense_ws holds two [B, max width] ping-pong rows.
static int run_dense(rmu_encoder* e, const SplitOperand& h, const int* cu, int B, int pool_mode, bool compact, int normalize,
                     float* out, cudaStream_t st) {
    const size_t half = static_cast<size_t>(B) * *std::max_element(e->dense_dims.begin(), e->dense_dims.end());
    int rc = grow(e->dense_ws, 2 * half * sizeof(float));
    if (rc != RMU_OK) return rc;
    float* buf[2] = {e->dense_ws.as<float>(), e->dense_ws.as<float>() + half};
    rc = launch_pool(h.hi, h.lo, cu, B, e->cfg.hidden, pool_mode, 0, compact, buf[0], st);
    const int n = static_cast<int>(e->dense_w.size());
    for (int l = 0; l < n && rc == RMU_OK; ++l) {
        const bool last = l == n - 1;
        rc = launch_dense(buf[l & 1], B, e->dense_dims[l], e->dense_dims[l + 1], e->dense_w[l], e->dense_b[l], e->dense_act[l],
                          last ? normalize : 0, last ? out : buf[(l + 1) & 1], st);
    }
    return rc;
}

// DeBERTa: grow the position terms' workspace to fit a call (qrows query rows, T keys)
static int ensure_position_ws(rmu_encoder* e, int qrows, int T, int max_seqlen) {
    const size_t floats = position_ws_floats(e->cidx_h.data(), e->cfg.max_pos - 1, max_seqlen, qrows, T, e->cfg.heads);
    return grow(e->pos_ws, floats * sizeof(float));
}

// the activation workspace for T tokens in B sequences, in the shape the create path recorded on the handle
static int ensure_tokens(rmu_encoder* e, int T, int B) {
    if (T <= e->tok_cap && B + 1 <= e->seq_cap) return RMU_OK;
    RMU_CUDA(cudaDeviceSynchronize());
    free_acts(e);
    const int H = e->cfg.hidden, F = e->cfg.ffn;
    const int cap = static_cast<int>(token_rows(T)), scap = static_cast<int>(seq_rows(B));
    // zero-filled: the GEMMs read A rows past a call's T (their outputs are clipped)
    auto planes = [&](SplitOperand* op, int rows, int cols) -> int {
        __half *hi = nullptr, *lo = nullptr;
        int rc = dev_alloc(e->act_allocs, &hi, static_cast<size_t>(rows) * cols);
        if (rc == RMU_OK) rc = dev_alloc(e->act_allocs, &lo, static_cast<size_t>(rows) * cols);
        if (rc != RMU_OK) return rc;
        RMU_CUDA(cudaMemset(hi, 0, static_cast<size_t>(rows) * cols * sizeof(__half)));
        RMU_CUDA(cudaMemset(lo, 0, static_cast<size_t>(rows) * cols * sizeof(__half)));
        return make_split_operand(op, hi, lo, rows, cols);
    };
    int rc = planes(&e->X, cap, H);
    if (rc == RMU_OK) rc = planes(&e->CTX, cap, e->ctx_w);
    if (rc == RMU_OK && e->has_x1) rc = planes(&e->X1, cap, H);
    if (rc == RMU_OK) rc = planes(&e->FF, cap, F);
    if (rc == RMU_OK) rc = planes(&e->QKVP, cap, e->qkv_w);
    if (rc == RMU_OK && e->has_qkvf) rc = dev_alloc(e->act_allocs, &e->QKVF, static_cast<size_t>(cap) * e->qkv_w);
    if (rc == RMU_OK) rc = dev_alloc(e->act_allocs, &e->PRE, static_cast<size_t>(cap) * H);
    if (e->has_cls_rows) {
        // one row per sequence: B exceeds T when sequences are empty
        if (rc == RMU_OK) rc = planes(&e->X_cls, scap, H);
        if (rc == RMU_OK) rc = planes(&e->Q_cls, scap, H);
        if (rc == RMU_OK) rc = planes(&e->CTX_cls, scap, H);
        if (rc == RMU_OK) rc = planes(&e->X1_cls, scap, H);
        if (rc == RMU_OK) rc = planes(&e->FF_cls, scap, F);
        if (rc == RMU_OK) rc = dev_alloc(e->act_allocs, &e->PRE_cls, static_cast<size_t>(scap) * H);
    }
    // the adapter's bottleneck activations reuse the FF planes (adapter_dim <= ffn)
    const int A = e->cfg.adapter_dim;
    if (rc == RMU_OK && A > 0) rc = make_split_operand(&e->FFA, e->FF.hi, e->FF.lo, cap, A);
    if (rc == RMU_OK && A > 0) rc = make_split_operand(&e->FFA_cls, e->FF_cls.hi, e->FF_cls.lo, scap, A);
    if (rc == RMU_OK && e->has_posi) rc = dev_alloc(e->act_allocs, &e->POSI, cap);
    if (rc != RMU_OK) { free_acts(e); return rc; }
    e->tok_cap = cap;
    e->seq_cap = scap;
    return RMU_OK;
}

// X-MOD's language adapter (adapter_dim > 0), between the FFN output and the layer's last LayerNorm.  pre [M, H] holds
// y = W2 ffn + b2 + x1 on entry and z on exit: h = LN2(y) goes into the x1 planes (free once the FFN-out GEMM has read
// its residual), then z = D2 gelu(D1 h + d1) + d2 + h through the ffa planes; the caller applies LN2 to z, the same
// gamma and beta again (adapter_reuse_layer_norm).  Every step computes a row from that row alone.
static int run_adapter(rmu_encoder* e, const EncLayer& L, int M, float* pre, const SplitOperand& x1, const SplitOperand& ffa,
                       cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, A = c.adapter_dim;
    int rc = launch_layernorm(pre, M, H, L.ln2g, L.ln2b, c.ln_eps, x1.hi, x1.lo, st);
    if (rc != RMU_OK) return rc;
    GemmParams g{};
    g.M = M; g.N = A; g.K = H; g.bias = L.d1; g.out_hi = ffa.hi; g.out_lo = ffa.lo;
    rc = launch_gemm(GEMM_BIAS_GELU_SPLIT, x1, L.D1, g, e->sms, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = M; g.N = H; g.K = A; g.bias = L.d2; g.out_f32 = pre; g.res_hi = x1.hi; g.res_lo = x1.lo;
    return launch_gemm(GEMM_BIAS_RESID_F32, ffa, L.D2, g, e->sms, st);
}

// The planes a post-LN layer runs on after its QKV projection: every token row (X, CTX, X1, FF, FFA, PRE) or one row
// per sequence (the _cls set of run_last_layer_cls).  x is the layer's input and, at the end, its output.
struct PostLnActs {
    const SplitOperand &x, &ctx, &x1, &ff, &ffa;
    float* pre;
};

// the layer's attention -> a.ctx: DeBERTa's disentangled attention when the model has position buckets, else E2 (with
// the relative bias table and, full rows only, the key limit nkeys).  cls_q non-null: the query rows are the CLS rows'
// compact q planes.
static int run_layer_attention(rmu_encoder* e, const EncLayer& L, const SplitOperand* cls_q, const int32_t* cu, int B,
                               int T, int max_seqlen, const SplitOperand& ctx, cudaStream_t st,
                               const int32_t* nkeys = nullptr) {
    const rmu_bert_config& c = e->cfg;
    const __half* q_hi = cls_q ? cls_q->hi : nullptr;
    const __half* q_lo = cls_q ? cls_q->lo : nullptr;
    if (e->ext.position_buckets > 0) {
        int rc = ensure_position_ws(e, cls_q ? B : T, T, max_seqlen);
        if (rc != RMU_OK) return rc;
        return run_disentangled_attention(e->QKVP.hi, e->QKVP.lo, q_hi, q_lo, cu, B, T, c.hidden, c.heads, max_seqlen,
                                          L.pos_hi, L.pos_lo, e->cidx, e->cidx_h.data(), c.max_pos - 1,
                                          e->pos_ws.as<float>(), ctx.hi, ctx.lo, st);
    }
    return launch_attention(e->QKVP.hi, e->QKVP.lo, q_hi, q_lo, cu, B, c.hidden, c.heads, max_seqlen, ctx.hi, ctx.lo, st,
                            e->rel, nkeys);
}

// a post-LN layer after its attention, on M rows: pre = ctx Wo^T + bo + x; x1 = LN1(pre); ff = gelu(x1 W1^T + b1);
// pre = ff W2^T + b2 + x1; X-MOD's adapter; x = LN2(pre)
static int run_post_ln_tail(rmu_encoder* e, const EncLayer& L, int M, const PostLnActs& a, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, F = c.ffn;
    GemmParams g{};
    g.M = M; g.N = H; g.K = H; g.bias = L.bo; g.out_f32 = a.pre; g.res_hi = a.x.hi; g.res_lo = a.x.lo;
    int rc = launch_gemm(GEMM_BIAS_RESID_F32, a.ctx, L.Wo, g, e->sms, st);
    if (rc != RMU_OK) return rc;
    rc = launch_layernorm(a.pre, M, H, L.ln1g, L.ln1b, c.ln_eps, a.x1.hi, a.x1.lo, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = M; g.N = F; g.K = H; g.bias = L.b1; g.out_hi = a.ff.hi; g.out_lo = a.ff.lo;
    rc = launch_gemm(GEMM_BIAS_GELU_SPLIT, a.x1, L.W1, g, e->sms, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = M; g.N = H; g.K = F; g.bias = L.b2; g.out_f32 = a.pre; g.res_hi = a.x1.hi; g.res_lo = a.x1.lo;
    rc = launch_gemm(GEMM_BIAS_RESID_F32, a.ff, L.W2, g, e->sms, st);
    if (rc != RMU_OK) return rc;
    if (c.adapter_dim > 0) {
        rc = run_adapter(e, L, M, a.pre, a.x1, a.ffa, st);
        if (rc != RMU_OK) return rc;
    }
    return launch_layernorm(a.pre, M, H, L.ln2g, L.ln2b, c.ln_eps, a.x.hi, a.x.lo, st);
}

// The last layer when only the CLS rows leave the encoder (classifier head, CLS pooling).  The CLS query attends to
// every key, so K and V are projected for all T rows, into the k | v columns of QKVP; everything else runs on row cu[b]
// of each sequence alone, gathered into row b of the compact planes, and leaves that row's hidden state in e->X_cls.
// Every kernel computes a row from that row's inputs alone with a fixed per-element order (E1 whatever the grid, E2 row 0
// whatever the other query rows, ln_kernel one warp per row), so those rows are bit-identical to the full layer's.
static int run_last_layer_cls(rmu_encoder* e, const EncLayer& L, const int32_t* cu, int B, int T, int max_seqlen,
                              float qscale, cudaStream_t st) {
    const int H = e->cfg.hidden;
    GemmParams g{};
    g.M = T; g.N = 2 * H; g.K = H; g.bias = L.bqkv + H;
    g.out_hi = e->QKVP.hi + H; g.out_lo = e->QKVP.lo + H; g.out_ld = 3 * H; g.qcols = 0; g.qscale = 1.0f;
    int rc = launch_gemm(GEMM_BIAS_SPLIT_QSCALE, e->X, e->last_wkv, g, e->sms, st);
    if (rc != RMU_OK) return rc;
    rc = launch_gather_cls_rows(e->X.hi, e->X.lo, cu, B, H, e->X_cls.hi, e->X_cls.lo, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = B; g.N = H; g.K = H; g.bias = L.bqkv; g.out_hi = e->Q_cls.hi; g.out_lo = e->Q_cls.lo; g.qcols = H; g.qscale = qscale;
    rc = launch_gemm(GEMM_BIAS_SPLIT_QSCALE, e->X_cls, e->last_wq, g, e->sms, st);
    if (rc == RMU_OK) rc = run_layer_attention(e, L, &e->Q_cls, cu, B, T, max_seqlen, e->CTX_cls, st);
    if (rc != RMU_OK) return rc;
    return run_post_ln_tail(e, L, B, {e->X_cls, e->CTX_cls, e->X1_cls, e->FF_cls, e->FFA_cls, e->PRE_cls}, st);
}

// ModernBERT's pre-LN stack (every layer in full): leaves final_norm of the residual stream in e->X.  The residual stream
// is never normalised, so it stays fp32, in e->PRE, updated in place by the fp32-residual epilogue:
//   x = LN_emb(tok_embeddings[id])                      (embed_ln_kernel with zero position / token-type rows)
//   per layer: a = (l == 0 ? x : LN_a(x)); x += Wo attn(rope(Wqkv a)); x += Wo2 geglu(Wi LN_m(x))
//   out = LN_final(x)
// Global layers (window 0) attend to the whole sequence with the rope tables of global_rope_theta, local ones to
// |i - j| <= window with those of local_rope_theta.
static int run_modernbert(rmu_encoder* e, const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T,
                          int max_seqlen, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, F = c.ffn, DH = H / c.heads;
    int rc = ensure_tokens(e, T, B);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaStreamWaitEvent(st, e->ws_done, 0));    // the activation workspace is shared by all callers
    rc = launch_seq_positions(cu, B, T, e->POSI, st);
    // one zero row for both the position and the token-type table: (w + 0) + 0 == w
    if (rc == RMU_OK)
        rc = launch_embed_ln(ids, type_ids, cu, B, T, H, c.vocab_size, 1, 1, e->word, e->pos, e->typ, e->eg, e->eb, c.ln_eps,
                             e->X.hi, e->X.lo, st);
    if (rc == RMU_OK) rc = launch_join_planes(e->X.hi, e->X.lo, static_cast<size_t>(T) * H, e->PRE, st);
    if (rc != RMU_OK) return rc;
    const float qscale = 1.4426950408889634f / sqrtf(static_cast<float>(DH));
    for (int l = 0; l < c.layers; ++l) {
        const EncLayer& L = e->layers[l];
        if (l > 0) {
            rc = launch_layernorm(e->PRE, T, H, L.ln1g, L.ln1b, c.ln_eps, e->X.hi, e->X.lo, st);
            if (rc != RMU_OK) return rc;
        }
        const int tab = L.window > 0 ? 1 : 0;
        GemmParams g{};
        g.M = T; g.N = 3 * H; g.K = H; g.bias = L.bqkv;
        g.out_hi = e->QKVP.hi; g.out_lo = e->QKVP.lo; g.qcols = H; g.qscale = qscale;
        g.pos = e->POSI; g.rope_cos = e->rope_cos[tab]; g.rope_sin = e->rope_sin[tab]; g.rope_hd = DH; g.rope_rows = c.max_pos;
        rc = launch_gemm(GEMM_BIAS_SPLIT_ROPE, e->X, L.Wqkv, g, e->sms, st);
        if (rc == RMU_OK)
            rc = launch_attention(e->QKVP.hi, e->QKVP.lo, nullptr, nullptr, cu, B, H, c.heads, max_seqlen, e->CTX.hi,
                                  e->CTX.lo, st, nullptr, nullptr, nullptr, L.window);
        if (rc != RMU_OK) return rc;
        g = GemmParams{};
        g.M = T; g.N = H; g.K = H; g.bias = L.bo; g.out_f32 = e->PRE; g.res_f32 = e->PRE;
        rc = launch_gemm(GEMM_BIAS_RESF32_F32, e->CTX, L.Wo, g, e->sms, st);
        if (rc == RMU_OK) rc = launch_layernorm(e->PRE, T, H, L.ln2g, L.ln2b, c.ln_eps, e->X1.hi, e->X1.lo, st);
        if (rc != RMU_OK) return rc;
        g = GemmParams{};
        g.M = T; g.N = 2 * F; g.K = H; g.bias = L.b1; g.out_hi = e->FF.hi; g.out_lo = e->FF.lo;
        rc = launch_gemm(GEMM_BIAS_GEGLU_SPLIT, e->X1, L.W1, g, e->sms, st);
        if (rc != RMU_OK) return rc;
        g = GemmParams{};
        g.M = T; g.N = H; g.K = F; g.bias = L.b2; g.out_f32 = e->PRE; g.res_f32 = e->PRE;
        rc = launch_gemm(GEMM_BIAS_RESF32_F32, e->FF, L.W2, g, e->sms, st);
        if (rc != RMU_OK) return rc;
    }
    return launch_layernorm(e->PRE, T, H, e->fng, e->fnb, c.ln_eps, e->X.hi, e->X.lo, st);
}

// the encoder stack: leaves the last hidden state in e->X (split planes), or with cls_only that of the CLS rows alone in
// e->X_cls (row b = sequence b; e->X then holds the input of the last layer).  nkeys ([B] device int32, not with
// cls_only): every layer's attention keys of sequence b stop at row nkeys[b] (ColBERT's [MASK] query padding).
static int run_encoder(rmu_encoder* e, const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T,
                       int max_seqlen, bool cls_only, cudaStream_t st, const int32_t* nkeys = nullptr) {
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, DH = H / c.heads;
    // the last position a sequence can reach is its length - 1 plus the offset (2 with padding-offset positions)
    const int pos_offset = c.position_mode == RMU_POS_OFFSET ? kPadId + 1 : 0;
    if (max_seqlen + pos_offset > c.max_pos) {
        set_error(pos_offset ? "sequence longer than max_position_embeddings - 2 (positions start after the padding index)"
                             : "sequence longer than max_position_embeddings");
        return RMU_ERR_ARG;
    }
    if (e->modern) return run_modernbert(e, ids, type_ids, cu, B, T, max_seqlen, st);
    int rc = ensure_tokens(e, T, B);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaStreamWaitEvent(st, e->ws_done, 0));    // the activation workspace is shared by all callers
    rc = launch_embed_ln(ids, type_ids, cu, B, T, H, c.vocab_size, c.max_pos, c.type_vocab, e->word, e->pos, e->typ, e->eg,
                         e->eb, c.ln_eps, e->X.hi, e->X.lo, st, c.position_mode);
    if (rc != RMU_OK) return rc;
    // q (scaled by 1/sqrt(dh), DeBERTa's three score terms by 1/sqrt(3 dh)), k, v leave the GEMM as split fp16 planes:
    // attention does no conversions (the softmax runs in base 2: q also carries log2(e))
    const float scale = 1.0f / sqrtf(static_cast<float>(e->ext.position_buckets > 0 ? 3 * DH : DH));
    const float qscale = scale * 1.4426950408889634f;
    if (cls_only && c.layers == 0) return launch_gather_cls_rows(e->X.hi, e->X.lo, cu, B, H, e->X_cls.hi, e->X_cls.lo, st);
    for (int l = 0; l < c.layers; ++l) {
        EncLayer& L = e->layers[l];
        if (cls_only && l == c.layers - 1) return run_last_layer_cls(e, L, cu, B, T, max_seqlen, qscale, st);
        GemmParams g{};
        g.M = T; g.N = 3 * H; g.K = H; g.bias = L.bqkv;
        g.out_hi = e->QKVP.hi; g.out_lo = e->QKVP.lo; g.qcols = H; g.qscale = qscale;
        rc = launch_gemm(GEMM_BIAS_SPLIT_QSCALE, e->X, L.Wqkv, g, e->sms, st);
        if (rc == RMU_OK) rc = run_layer_attention(e, L, nullptr, cu, B, T, max_seqlen, e->CTX, st, nkeys);
        if (rc == RMU_OK) rc = run_post_ln_tail(e, L, T, {e->X, e->CTX, e->X1, e->FF, e->FFA, e->PRE}, st);
        if (rc != RMU_OK) return rc;
    }
    return RMU_OK;
}

// projection `which` (0 Wqkv, 1 Wo, 2 W1, 3 W2) of a decoder layer, C = A W^T with E1's epilogue `mode`.  Split
// planes: E1.  NF4 with `gemv` (a decode step, or the prefill of a one-token prompt): the decode GEMV, one row or
// several; otherwise the weight dequantised into the scratch planes, then E1 on them (the scratch is reused by the
// next projection in stream order).  The caller chooses by the prompt, not by M: a batched prefill's chunk of one
// row takes the path the whole prompt's prefill takes.
static SplitOperand EncLayer::* const kDecoderSplit[4] = {&EncLayer::Wqkv, &EncLayer::Wo, &EncLayer::W1, &EncLayer::W2};

static int decoder_gemm(rmu_encoder* e, int mode, const SplitOperand& A, const EncLayer& L, int which, const GemmParams& g,
                        bool gemv, cudaStream_t st) {
    if (!e->nf4) return launch_gemm(mode, A, L.*kDecoderSplit[which], g, e->sms, st);
    const Nf4Weight& W = L.nf4[which];
    if (gemv)
        return g.M == 1 ? launch_nf4_gemv(mode, A.hi, A.lo, W, g, e->sms, st)
                        : launch_nf4_gemv_rows(mode, A.hi, A.lo, W, g, e->sms, st);
    const int rc = launch_nf4_dequantize(W.codes, W.absmax, static_cast<int64_t>(W.rows) * W.cols, e->nf4_hi, st);
    return rc != RMU_OK ? rc : launch_gemm(mode, A, e->nf4_op[which], g, e->sms, st);
}

// one decoder layer up to its attention inputs: X = split(w_in RMS(h)); QKVF = X Wqkv^T (fp32); QKVP = the q / k step
static int qwen3_attention_inputs(rmu_encoder* e, const EncLayer& L, int T, bool gemv, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int nh = c.heads, kv = e->qext.kv_heads, NQKV = (nh + 2 * kv) * kQwenHD;
    const float qscale = 1.4426950408889634f / sqrtf(static_cast<float>(kQwenHD));
    int rc = launch_rms_split(e->PRE, T, c.hidden, L.ln1g, c.ln_eps, e->X.hi, e->X.lo, e->range_flag, st);
    if (rc != RMU_OK) return rc;
    GemmParams g{};
    g.M = T; g.N = NQKV; g.K = c.hidden; g.bias = e->zeros; g.out_f32 = e->QKVF;
    rc = decoder_gemm(e, GEMM_BIAS_F32, e->X, L, 0, g, gemv, st);
    if (rc != RMU_OK) return rc;
    return launch_qk_norm_rope(e->QKVF, T, nh, kv, e->POSI, L.qn, L.kn, c.ln_eps, qscale, e->rope_cos[0], e->rope_sin[0],
                               c.max_pos, e->QKVP.hi, e->QKVP.lo, e->range_flag, st);
}

// one decoder layer after its attention, on M rows: h += CTX Wo^T (in place); X = split(w_post RMS(h)); FF =
// split(silu(X Wgate^T) * (X Wup^T)); h += FF Wdown^T
static int qwen3_layer_tail(rmu_encoder* e, const EncLayer& L, int M, bool gemv, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, F = c.ffn, QD = c.heads * kQwenHD;
    GemmParams g{};
    g.M = M; g.N = H; g.K = QD; g.bias = e->zeros; g.out_f32 = e->PRE; g.res_f32 = e->PRE;
    int rc = decoder_gemm(e, GEMM_BIAS_RESF32_F32, e->CTX, L, 1, g, gemv, st);
    if (rc == RMU_OK) rc = launch_rms_split(e->PRE, M, H, L.ln2g, c.ln_eps, e->X.hi, e->X.lo, e->range_flag, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = M; g.N = 2 * F; g.K = H; g.bias = e->zeros; g.out_hi = e->FF.hi; g.out_lo = e->FF.lo; g.range_flag = e->range_flag;
    rc = decoder_gemm(e, GEMM_BIAS_SWIGLU_SPLIT, e->X, L, 2, g, gemv, st);
    if (rc != RMU_OK) return rc;
    g = GemmParams{};
    g.M = M; g.N = H; g.K = F; g.bias = e->zeros; g.out_f32 = e->PRE; g.res_f32 = e->PRE;
    return decoder_gemm(e, GEMM_BIAS_RESF32_F32, e->FF, L, 3, g, gemv, st);
}

// A KV cache in kv_append_kernel's layout, [layers][K hi | K lo | V hi | V lo][kv_heads][cap][128]: the handle's own
// (handle_kv) or a decode session's
struct KvView {
    __half* base = nullptr;
    int cap = 0;
};

static KvView handle_kv(rmu_encoder* e) { return KvView{e->kv_cache.as<__half>(), e->kv_cap}; }

// layer l's K / V planes in the cache v
static __half* kv_layer(const rmu_encoder* e, const KvView& v, int l) {
    return v.base + static_cast<size_t>(l) * 4 * e->qext.kv_heads * v.cap * kQwenHD;
}

static __half* kv_layer(rmu_encoder* e, int l) { return kv_layer(e, handle_kv(e), l); }

// grow the handle's KV cache to hold at least cap positions
static int ensure_kv(rmu_encoder* e, const std::string& fn, int cap) {
    if (cap <= e->kv_cap) return RMU_OK;
    e->kv_cap = 0;                                      // until grow succeeds: it may free the old cache first
    const int rc = grow(e->kv_cache, static_cast<size_t>(e->cfg.layers) * 4 * e->qext.kv_heads * cap * kQwenHD * sizeof(__half));
    if (rc != RMU_OK) set_error(fn + ": the KV cache for " + std::to_string(cap) + " positions: " + rmu_last_error());
    else e->kv_cap = cap;
    return rc;
}

// the rmu_decoder_* entry points run on decoder handles only
static int check_decoder(const rmu_encoder* e, const std::string& fn) {
    if (e->qwen && !e->has_head) return RMU_OK;
    set_error(fn + ": the encoder must come from rmu_encoder_create_qwen3 without a head or from rmu_encoder_create_llama");
    return RMU_ERR_ARG;
}

// a handle whose NF4 conversion failed part-way, or one built layer by layer whose layers are not all loaded, runs
// nothing
static int check_nf4_intact(const rmu_encoder* e, const std::string& fn) {
    if (e->by_layer && e->layers_loaded < e->cfg.layers) {
        set_error(fn + ": layer " + std::to_string(e->layers_loaded) + " of " + std::to_string(e->cfg.layers) +
                  " is not loaded (rmu_decoder_load_layer_nf4)");
        return RMU_ERR_ARG;
    }
    if (!e->nf4_broken) return RMU_OK;
    set_error(fn + ": the handle's NF4 conversion failed part-way (rmu_decoder_quantize_nf4); destroy it");
    return RMU_ERR_ARG;
}

// the generation entry points run on an intact decoder handle with an LM head
static int check_generator(const rmu_encoder* e, const std::string& fn) {
    int rc = check_decoder(e, fn);
    if (rc != RMU_OK) return rc;
    if (!e->has_lm_head) { set_error(fn + ": no LM head is attached (rmu_decoder_set_lm_head)"); return RMU_ERR_ARG; }
    return check_nf4_intact(e, fn);
}

// the prompts b < B, ids_h[cu_h[b] .. cu_h[b + 1]), a generation entry point refuses before any CUDA call
static int check_prompts(const rmu_encoder* e, const std::string& fn, const int32_t* ids_h, const int32_t* cu_h, int B) {
    const rmu_bert_config& c = e->cfg;
    for (int b = 0; b < B; ++b) {
        const int T = cu_h[b + 1] - cu_h[b];
        if (T <= 0 || cu_h[b] < 0) { set_error(fn + ": prompt " + std::to_string(b) + " is empty"); return RMU_ERR_ARG; }
        if (T >= c.max_pos) {
            set_error(fn + ": a prompt of " + std::to_string(T) + " tokens leaves no position for a new token " +
                      "(max_position_embeddings " + std::to_string(c.max_pos) + ")");
            return RMU_ERR_ARG;
        }
        for (int i = cu_h[b]; i < cu_h[b + 1]; ++i)
            if (ids_h[i] < 0 || ids_h[i] >= c.vocab_size) { set_error(fn + ": token id out of range"); return RMU_ERR_ARG; }
    }
    return RMU_OK;
}

// Qwen3's layers (the header's formula): leaves the residual stream h, before the final norm, in e->PRE [T, H] fp32.
// Per layer: the attention inputs (above); CTX = causal GQA attention; then qwen3_layer_tail.  With attn_last (the span
// attention), the last layer stops at its attention inputs, which QKVP then holds.  With to_cache (one sequence, the
// prefill of rmu_decoder_generate), each layer's k and v rows also go to the KV cache at positions 0 .. T - 1.
// The range flag is cleared first; the caller reads it (qwen3_check_range) before it writes an output.
static int run_qwen3(rmu_encoder* e, const int32_t* ids, const int32_t* cu, int B, int T, int max_seqlen, cudaStream_t st,
                     bool attn_last = false, bool to_cache = false) {
    const rmu_bert_config& c = e->cfg;
    if (max_seqlen > c.max_pos) { set_error("sequence longer than max_position_embeddings"); return RMU_ERR_ARG; }
    int rc = check_nf4_intact(e, e->llama ? "Llama forward" : "Qwen3 forward");
    if (rc != RMU_OK) return rc;
    const int H = c.hidden, nh = c.heads, kv = e->qext.kv_heads;
    rc = ensure_tokens(e, T, B);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaStreamWaitEvent(st, e->ws_done, 0));    // the activation workspace is shared by all callers
    RMU_CUDA(cudaMemsetAsync(e->range_flag, 0, sizeof(int), st));
    rc = launch_seq_positions(cu, B, T, e->POSI, st);
    if (rc == RMU_OK) rc = launch_embed_rows(ids, T, H, c.vocab_size, e->word, e->PRE, st);
    if (rc != RMU_OK) return rc;
    for (int l = 0; l < c.layers; ++l) {
        const EncLayer& L = e->layers[l];
        rc = qwen3_attention_inputs(e, L, T, T == 1, st);
        if (rc != RMU_OK || (attn_last && l == c.layers - 1)) return rc;
        if (to_cache) rc = launch_kv_append(e->QKVP.hi, e->QKVP.lo, T, nh, kv, 0, e->kv_cap, kv_layer(e, l), st);
        if (rc == RMU_OK)
            rc = launch_attention_causal(e->QKVP.hi, e->QKVP.lo, cu, B, nh, kv, max_seqlen, e->CTX.hi, e->CTX.lo, st);
        if (rc == RMU_OK) rc = qwen3_layer_tail(e, L, T, T == 1, st);
        if (rc != RMU_OK) return rc;
    }
    return RMU_OK;
}

// whether the range flag of the split kernels is raised, cleared again when it is (synchronises st)
static int read_range(rmu_encoder* e, bool* raised, cudaStream_t st) {
    int flag = 0;
    RMU_CUDA(cudaMemcpyAsync(&flag, e->range_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    *raised = flag != 0;
    if (flag) RMU_CUDA(cudaMemsetAsync(e->range_flag, 0, sizeof(int), st));
    return RMU_OK;
}

// reads the range flag of run_qwen3's split kernels (synchronises st): RMU_ERR_RANGE when an activation left fp16's range
static int qwen3_check_range(rmu_encoder* e, cudaStream_t st) {
    bool raised = false;
    const int rc = read_range(e, &raised, st);
    if (rc != RMU_OK || !raised) return rc;
    set_error(std::string(e->llama ? "Llama" : "Qwen3") + " forward: an activation entering a GEMM or attention left the fp16 range of the split planes "
              "(|x| > 65504); the encoder cannot compute this model's activations for this input");
    return RMU_ERR_RANGE;
}

// One prefill run of rmu_decoder_generate_batch over B sequences of T token rows in all (cu [B + 1]): each row's
// position and cache row offset are in e->POSI and shift (uploaded by the caller), so token t of sequence b is at
// position P + t and its k / v go to cache row P + t + shift; attention is attention_causal_kernel's cached form
// (PrefixKeys), keys below P from the shared prefix rows.  The range flag is not cleared: the caller clears it once
// per call.  The activation workspace must already hold T rows (ensure_tokens).
static int run_batch_prefill(rmu_encoder* e, const KvView& kvv, const int32_t* ids, const int32_t* cu, const int* shift,
                             int B, int T, int max_own, int P, bool gemv, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int nh = c.heads, kv = e->qext.kv_heads;
    int rc = launch_embed_rows(ids, T, c.hidden, c.vocab_size, e->word, e->PRE, st);
    for (int l = 0; l < c.layers && rc == RMU_OK; ++l) {
        const EncLayer& L = e->layers[l];
        rc = qwen3_attention_inputs(e, L, T, gemv, st);
        if (rc == RMU_OK) rc = launch_kv_append(e->QKVP.hi, e->QKVP.lo, T, nh, kv, 0, kvv.cap, kv_layer(e, kvv, l), st, e->POSI, shift);
        PrefixKeys pk;
        pk.kv = kv_layer(e, kvv, l);
        pk.shift = shift;
        pk.cap = kvv.cap;
        pk.P = P;
        if (rc == RMU_OK) rc = launch_attention_cached(e->QKVP.hi, e->QKVP.lo, cu, B, nh, kv, max_own, pk, e->CTX.hi, e->CTX.lo, st);
        if (rc == RMU_OK) rc = qwen3_layer_tail(e, L, T, gemv, st);
    }
    return rc;
}

// The host rows of one run_batch_prefill: tokens from .. T_b - 1 of each prompt b = seqs[i] (ids_h[cu_h[b] ..),
// T_b = cu_h[b + 1] - cu_h[b]), token t at position t and cache row t + shift[i]; cu [seqs + 1] over the rows
struct PrefillRows {
    std::vector<int> ids, cu{0}, shift, pos;
    int max_own = 0;
};

static PrefillRows prefill_rows(const int32_t* ids_h, const int32_t* cu_h, const std::vector<int>& seqs, int from,
                                const std::vector<int>& shift) {
    PrefillRows pr;
    for (size_t i = 0; i < seqs.size(); ++i) {
        const int b = seqs[i], n = cu_h[b + 1] - cu_h[b] - from;
        for (int t = from; t < from + n; ++t) {
            pr.ids.push_back(ids_h[cu_h[b] + t]);
            pr.pos.push_back(t);
            pr.shift.push_back(shift[i]);
        }
        pr.cu.push_back(pr.cu.back() + n);
        pr.max_own = std::max(pr.max_own, n);
    }
    return pr;
}

// the last row of each sequence i of a prefill (cu) from e->PRE to row at[i] of last [., H] (at null: row i)
static int gather_last(rmu_encoder* e, const std::vector<int>& cu, const int* at, float* last, cudaStream_t st) {
    const size_t H = e->cfg.hidden;
    for (size_t i = 0; i + 1 < cu.size(); ++i)
        RMU_CUDA(cudaMemcpyAsync(last + (at ? at[i] : i) * H, e->PRE + (cu[i + 1] - 1) * H, H * 4, cudaMemcpyDeviceToDevice, st));
    return RMU_OK;
}

// The prefill runs of B prompts of Tb tokens: an NF4 handle's one-token prompts one by one (on the GEMV their own
// prefill takes), then the others together
static std::vector<std::vector<int>> prefill_groups(const rmu_encoder* e, const std::vector<int>& Tb) {
    std::vector<std::vector<int>> groups;
    std::vector<int> rest;
    for (int b = 0; b < static_cast<int>(Tb.size()); ++b) {
        if (e->nf4 && Tb[b] == 1) groups.push_back({b});
        else rest.push_back(b);
    }
    if (!rest.empty()) groups.push_back(rest);
    return groups;
}

// the sampling settings rmu_decoder_generate and rmu_debug_sample refuse, before any CUDA call
static int check_sampling(const std::string& fn, const rmu_sampling* s) {
    if (s->n_eos < 0 || s->n_eos > RMU_MAX_EOS || !(s->repetition_penalty > 0.f) || !std::isfinite(s->repetition_penalty)) {
        set_error(fn + ": n_eos must be 0 .. 8 and repetition_penalty a positive finite number");
        return RMU_ERR_ARG;
    }
    if (s->do_sample) {
        if (s->top_k < 1 || s->top_k > kSampleCap) {
            set_error(fn + ": top_k must be 1 .. 256 when sampling, got " + std::to_string(s->top_k));
            return RMU_ERR_UNSUPPORTED;
        }
        if (!(s->temperature > 0.f) || !std::isfinite(s->temperature) || !(s->top_p > 0.f && s->top_p <= 1.f)) {
            set_error(fn + ": temperature must be positive and finite and top_p in (0, 1] when sampling");
            return RMU_ERR_ARG;
        }
    }
    return RMU_OK;
}

static SampleArgs sample_args(const rmu_sampling& s) {
    return SampleArgs{s.do_sample ? 1 : 0, s.top_k, s.temperature, s.top_p, s.repetition_penalty};
}

// a prompt's presence bits: out [words] has bit i set for each id i among ids [n]
static void prompt_bits(const int32_t* ids, int n, size_t words, unsigned* out) {
    std::fill(out, out + words, 0u);
    for (int i = 0; i < n; ++i) out[ids[i] >> 5] |= 1u << (ids[i] & 31);
}

// a reply's status after its n-th token t, for a prompt of T tokens: RMU_GEN_LIVE, or why it stops
static int stop_status(const rmu_sampling& s, int t, int n, int max_new, int T, int max_pos) {
    for (int i = 0; i < s.n_eos; ++i)
        if (t == s.eos_ids[i]) return RMU_GEN_EOS;
    if (n == max_new) return RMU_GEN_MAX_NEW;
    if (T + n >= max_pos) return RMU_GEN_MAX_POS;
    return RMU_GEN_LIVE;
}

// One batched decode step's layers (rmu_decoder_generate_batch's steps, a prompt-lookup verify pass): M token rows
// ids [M] (device) at the positions in e->POSI (uploaded by the caller), row r's k / v into cache row pos[r] +
// shift[r] and its attention over keys [0, pos[r] + 1) with the DecRows prefix mapping P; maxn = the most keys of any
// row; part holds M * decode_part_floats(heads, maxn) floats.  The rows' hidden states are left in e->PRE.
static int run_decode_rows(rmu_encoder* e, const KvView& kvv, const int* ids, int M, const int* shift, int P, int maxn,
                           float* part, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int nh = c.heads, kv = e->qext.kv_heads;
    int rc = launch_embed_rows(ids, M, c.hidden, c.vocab_size, e->word, e->PRE, st);
    DecRows dr;
    dr.pos = e->POSI;
    dr.shift = shift;
    dr.P = P;
    dr.qld = static_cast<size_t>(nh + 2 * kv) * kQwenHD;
    for (int l = 0; l < c.layers && rc == RMU_OK; ++l) {
        const EncLayer& Ly = e->layers[l];
        rc = qwen3_attention_inputs(e, Ly, M, true, st);
        if (rc == RMU_OK) rc = launch_kv_append(e->QKVP.hi, e->QKVP.lo, M, nh, kv, 0, kvv.cap, kv_layer(e, kvv, l), st, e->POSI, shift);
        if (rc == RMU_OK)
            rc = launch_attention_decode(e->QKVP.hi, e->QKVP.lo, kv_layer(e, kvv, l), nh, kv, kvv.cap, maxn, part, e->CTX.hi,
                                         e->CTX.lo, st, M, dr);
        if (rc == RMU_OK) rc = qwen3_layer_tail(e, Ly, M, true, st);
    }
    return rc;
}

// The single-row decode step: the token id [1] (device) at position p through every layer, its k / v into cache row
// p of the handle's cache and its attention over keys [0, p + 1); part holds decode_part_floats(heads, p + 1) floats.
// The row's hidden state is left in e->PRE.
static int run_decode_step(rmu_encoder* e, const int* id, int p, float* part, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    const int nh = c.heads, kv = e->qext.kv_heads;
    set_int_kernel<<<1, 1, 0, st>>>(e->POSI, p);
    count_launch();
    RMU_CHECK_LAUNCH();
    int rc = launch_embed_rows(id, 1, c.hidden, c.vocab_size, e->word, e->PRE, st);
    for (int l = 0; l < c.layers && rc == RMU_OK; ++l) {
        const EncLayer& Ly = e->layers[l];
        rc = qwen3_attention_inputs(e, Ly, 1, true, st);
        if (rc == RMU_OK) rc = launch_kv_append(e->QKVP.hi, e->QKVP.lo, 1, nh, kv, p, e->kv_cap, kv_layer(e, l), st);
        if (rc == RMU_OK)
            rc = launch_attention_decode(e->QKVP.hi, e->QKVP.lo, kv_layer(e, l), nh, kv, e->kv_cap, p + 1, part, e->CTX.hi,
                                         e->CTX.lo, st);
        if (rc == RMU_OK) rc = qwen3_layer_tail(e, Ly, 1, true, st);
    }
    return rc;
}

// logits [M, V] = lm_head . (w_norm RMS(x)) for M fp32 hidden rows x [M, H]
static int run_lm_head(rmu_encoder* e, const float* x, int M, float* logits, cudaStream_t st) {
    const rmu_bert_config& c = e->cfg;
    int rc = launch_rms_split(x, M, c.hidden, e->fng, c.ln_eps, e->X.hi, e->X.lo, e->range_flag, st);
    if (rc != RMU_OK) return rc;
    ProfScope _ps(PROF_LM_HEAD, st);
    GemmParams gp{};
    gp.M = M; gp.N = c.vocab_size; gp.K = c.hidden; gp.bias = e->lm_zero; gp.out_f32 = logits;
    return launch_gemm(GEMM_BIAS_F32, e->X, e->lm_head, gp, e->sms, st);
}

constexpr int kMaxDrafts = RMU_MAX_GENERATE_BATCH - 1;   // a verify pass feeds at most 16 rows

// a drafter (prompt lookup, a draft model): up to k ids that may follow seq (the prompt and the tokens so far) -> out,
// their count, or a negative error code that fails the call
using Drafter = std::function<int(const std::vector<int32_t>& seq, int k, int32_t* out)>;

// the refusals of rmu_decoder_generate and its drafting forms, before any CUDA call
static int check_generate(rmu_encoder* e, const std::string& fn, const int32_t* ids_h, int T, const rmu_sampling* s) {
    const int cu_h[2] = {0, T};
    int rc = check_generator(e, fn);
    if (rc == RMU_OK) rc = check_prompts(e, fn, ids_h, cu_h, 1);
    if (rc == RMU_OK) rc = check_sampling(fn, s);
    return rc;
}

// The generation loop of rmu_decoder_generate and its drafting forms (DESIGN.md, "Prompt-lookup decoding").  The
// prefill's last row gives the first token; each later pass feeds the pending token at position p = T + n - 1 plus k
// drafts at p + 1 .. p + k, k = 0 .. kmax.  k = 0 is the single-row step.  k >= 1 is a verify pass: run_decode_rows on
// the k + 1 rows, row j sampling as sequential step n + j would (its own presence bits: the base plus drafts 1 .. j;
// Philox step n + j); t_0 is kept, t_j while t_{j - 1} equals draft j.  A verify pass that raises the range flag is
// redone as a k = 0 step at the same position, so RMU_ERR_RANGE means what it means without drafts.  The caller has
// passed check_generate and holds the handle's host_mu and mu.  n_drafted / n_kept (nullable): the drafts proposed and
// the drafts emitted as tokens.
static int generate_loop(rmu_encoder* e, const std::string& fn, const int32_t* ids_h, int T, const rmu_sampling* s,
                         uint64_t seed, int max_new_tokens, int kmax, const Drafter& draft, int32_t* out_h, int32_t* n_out,
                         float* logits_h, int32_t* n_passes, void* stream, int32_t* n_drafted = nullptr,
                         int32_t* n_kept = nullptr) {
    const int cu_h[2] = {0, T};
    int rc = RMU_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const rmu_bert_config& c = e->cfg;
    const int V = c.vocab_size, H = c.hidden, nh = c.heads;
    const int cap = std::min(T + max_new_tokens, c.max_pos);
    // gen_ws: logits [R, V] | presence [words] | tokens [R] | decode partials [R rows] and, for verify passes, presence
    // rows [R, words] | ints: ids [R] | shift [R] (zeros); R = kmax + 1
    const int R = kmax + 1, Rv = R > 1 ? R : 0;
    const size_t words = (static_cast<size_t>(V) + 31) / 32, part_f = decode_part_floats(nh, cap);
    float *logits, *part;
    unsigned *presence, *prow;
    int *tok, *ints;
    auto layout = [&](void* base) {
        Carve w(base);
        logits = w.take<float>(static_cast<size_t>(R) * V);
        presence = w.take<unsigned>(words);
        tok = w.take<int>(R);
        part = w.take<float>(R * part_f);
        prow = w.take<unsigned>(Rv * words);
        ints = w.take<int>(2 * Rv);
        return w.size;
    };
    rc = ensure_kv(e, fn, cap);
    if (rc == RMU_OK) rc = grow(e->gen_ws, layout(nullptr));
    if (rc == RMU_OK) rc = grow(e->d_ids, T * sizeof(int32_t), token_rows(T) * sizeof(int32_t));
    if (rc == RMU_OK && R > 1) rc = ensure_tokens(e, R, 1);
    if (rc != RMU_OK) return rc;
    layout(e->gen_ws.p);
    std::vector<unsigned> bits(words);
    prompt_bits(ids_h, T, words, bits.data());
    RMU_CUDA(cudaStreamWaitEvent(st, e->ws_done, 0));    // gen_ws is shared by all callers
    // pageable sources: each copy has taken its bytes when it returns
    RMU_CUDA(cudaMemcpyAsync(e->d_ids.p, ids_h, T * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(e->span_cu, cu_h, sizeof(cu_h), cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(presence, bits.data(), words * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    std::vector<int> hints(2 * static_cast<size_t>(R), 0), hpos(R), t_h(R);
    if (R > 1) RMU_CUDA(cudaMemcpyAsync(ints, hints.data(), hints.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    std::vector<int32_t> seq(ids_h, ids_h + T);          // the prompt and the tokens so far: what the drafter reads
    std::vector<float> staged(logits_h && R > 1 ? static_cast<size_t>(R) * V : 0);
    const SampleArgs sa = sample_args(*s);
    // the prefill writes the cache; its last row's hidden state gives the first token
    rc = run_qwen3(e, e->d_ids.as<int32_t>(), e->span_cu, 1, T, T, st, false, true);
    const float* last = e->PRE + static_cast<size_t>(T - 1) * H;
    int n = 0, passes = 0, drafted = 0, kept = 0;
    bool redo = false;                                     // the last verify pass raised the range flag
    while (rc == RMU_OK) {
        const int p = T + n - 1;
        int k = 0;
        if (n > 0 && kmax > 0 && !redo) {
            // a pass never writes past output index max_new_tokens - 1 or position max_pos - 1
            k = std::min({kmax, max_new_tokens - 1 - n, c.max_pos - 1 - T - n});
            if (k > 0) k = draft(seq, k, hints.data() + 1);
            if (k < 0) { rc = k; break; }
            drafted += k;
        }
        redo = false;
        int acc = 1;                                       // tokens this pass keeps: t_h[0 .. acc)
        if (k == 0) {
            if (n > 0) {
                // after a verify pass the pending token is the last kept row's, not tok[0]: it goes up through ints
                const int* pending = tok;
                if (kmax > 0) {
                    hints[0] = seq.back();
                    RMU_CUDA(cudaMemcpyAsync(ints, hints.data(), sizeof(int), cudaMemcpyHostToDevice, st));
                    pending = ints;
                }
                // the previous token at position p through every layer, its k / v into cache row p
                rc = run_decode_step(e, pending, p, part, st);
                last = e->PRE;
            }
            if (rc == RMU_OK) rc = run_lm_head(e, last, 1, logits, st);
            if (rc == RMU_OK && logits_h)
                RMU_CUDA(cudaMemcpyAsync(logits_h + static_cast<size_t>(n) * V, logits, static_cast<size_t>(V) * sizeof(float),
                                         cudaMemcpyDeviceToHost, st));
            if (rc == RMU_OK) rc = launch_sample(logits, V, presence, sa, -1.f, seed, static_cast<unsigned long long>(n), tok, st);
            if (rc != RMU_OK) break;
            RMU_CUDA(cudaMemcpyAsync(t_h.data(), tok, sizeof(int), cudaMemcpyDeviceToHost, st));
            rc = qwen3_check_range(e, st);        // synchronises st
            if (rc != RMU_OK) break;
        } else {
            // rows j = 0 .. k: token hints[j] (the pending token, then the drafts) at position p + j, cache row p + j
            const int M = k + 1;
            hints[0] = seq.back();
            for (int j = 0; j < M; ++j) hpos[j] = p + j;
            RMU_CUDA(cudaMemcpyAsync(ints, hints.data(), M * sizeof(int), cudaMemcpyHostToDevice, st));
            RMU_CUDA(cudaMemcpyAsync(e->POSI, hpos.data(), M * sizeof(int), cudaMemcpyHostToDevice, st));
            rc = launch_presence_rows(presence, words, ints, M, prow, st);
            if (rc == RMU_OK) rc = run_decode_rows(e, handle_kv(e), ints, M, ints + R, 0, p + M, part, st);
            if (rc == RMU_OK) rc = run_lm_head(e, e->PRE, M, logits, st);
            if (rc == RMU_OK && logits_h)
                RMU_CUDA(cudaMemcpyAsync(staged.data(), logits, static_cast<size_t>(M) * V * sizeof(float),
                                         cudaMemcpyDeviceToHost, st));
            SampleRows sr;
            sr.words = words;
            sr.row_step = true;
            if (rc == RMU_OK) rc = launch_sample(logits, V, prow, sa, -1.f, seed, static_cast<unsigned long long>(n), tok, st, M, sr);
            if (rc != RMU_OK) break;
            RMU_CUDA(cudaMemcpyAsync(t_h.data(), tok, M * sizeof(int), cudaMemcpyDeviceToHost, st));
            ++passes;
            rc = read_range(e, &redo, st);                 // synchronises st; a rejected draft's row may be the cause
            if (rc != RMU_OK || redo) continue;
            while (acc < M && t_h[acc - 1] == hints[acc]) ++acc;
            // the last kept row's bits are the base plus every kept token: the next base
            RMU_CUDA(cudaMemcpyAsync(presence, prow + static_cast<size_t>(acc - 1) * words, words * sizeof(unsigned),
                                     cudaMemcpyDeviceToDevice, st));
        }
        if (n > 0 && k == 0) ++passes;
        bool stop = false;
        for (int j = 0; j < acc && !stop; ++j) {
            if (k > 0 && logits_h)
                std::copy(staged.begin() + static_cast<size_t>(j) * V, staged.begin() + static_cast<size_t>(j + 1) * V,
                          logits_h + static_cast<size_t>(n) * V);
            out_h[n++] = t_h[j];
            seq.push_back(t_h[j]);
            kept += j > 0;
            stop = stop_status(*s, t_h[j], n, max_new_tokens, T, c.max_pos) != RMU_GEN_LIVE;
        }
        if (stop) break;
    }
    *n_out = n;
    if (n_passes) *n_passes = passes;
    if (n_drafted) *n_drafted = drafted;
    if (n_kept) *n_kept = kept;
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

static int check_batch(const rmu_encoder* e, const void* ids, const void* cu, int B, int T, const void* out) {
    if (!e || !ids || !cu || !out || B <= 0 || T <= 0) { set_error("encoder: bad argument"); return RMU_ERR_ARG; }
    return RMU_OK;
}

extern "C" {

int rmu_encoder_create(const rmu_bert_config* cfg, const float* const* w, int n_weights, int has_head, rmu_encoder** out) {
    return rmu_encoder_create_ex(cfg, nullptr, w, n_weights, has_head, out);
}

int rmu_encoder_create_ex(const rmu_bert_config* cfg, const rmu_encoder_ext* ext_in, const float* const* w, int n_weights,
                          int has_head, rmu_encoder** out) {
    if (!cfg || !w || !out) { set_error("rmu_encoder_create: bad argument"); return RMU_ERR_ARG; }
    const rmu_encoder_ext ext = ext_in ? *ext_in : rmu_encoder_ext{};
    const int H = cfg->hidden, F = cfg->ffn, L = cfg->layers;
    if (cfg->position_mode != RMU_POS_ABSOLUTE && cfg->position_mode != RMU_POS_OFFSET) {
        set_error("rmu_encoder_create: position_mode must be RMU_POS_ABSOLUTE (0) or RMU_POS_OFFSET (1)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (cfg->rel_buckets != 0 && cfg->rel_buckets != 32) {
        set_error("rmu_encoder_create: rel_buckets must be 0 (no relative position bias) or 32 (MPNet)");
        return RMU_ERR_UNSUPPORTED;
    }
    const int A = cfg->adapter_dim;
    if (A < 0 || A % 128 != 0 || A > F) {
        set_error("rmu_encoder_create: adapter_dim must be 0 (no adapter) or a multiple of 128 no larger than ffn");
        return RMU_ERR_UNSUPPORTED;
    }
    const int PB = ext.position_buckets, MRP = ext.max_relative_positions;
    if (ext.head_act != RMU_HEAD_TANH && ext.head_act != RMU_HEAD_GELU && ext.head_act != RMU_HEAD_RELU) {
        set_error("rmu_encoder_create: head_act must be RMU_HEAD_TANH (0), RMU_HEAD_GELU (1) or RMU_HEAD_RELU (2)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (ext.head_act == RMU_HEAD_RELU && PB != 0) {
        // DistilBERT's head; no model pairs it with disentangled attention
        set_error("rmu_encoder_create: head_act RMU_HEAD_RELU (DistilBERT's head) takes position_buckets 0");
        return RMU_ERR_UNSUPPORTED;
    }
    if (PB < 0 || (PB == 0 && MRP != 0) || PB > 4096) {
        set_error("rmu_encoder_create: position_buckets must be 0 (with max_relative_positions 0) or 1..4096");
        return RMU_ERR_UNSUPPORTED;
    }
    if (PB > 0 && (PB < 2 || MRP < PB / 2 + 2)) {
        set_error("rmu_encoder_create: position_buckets needs at least 2 buckets and max_relative_positions >= "
                  "position_buckets / 2 + 2");
        return RMU_ERR_UNSUPPORTED;
    }
    if (PB > 0 && (cfg->rel_buckets != 0 || A != 0 || cfg->heads <= 0 || H % cfg->heads != 0 || H / cfg->heads != 64)) {
        set_error("rmu_encoder_create: disentangled attention (position_buckets > 0) runs with head_dim 64, without "
                  "rel_buckets or an adapter");
        return RMU_ERR_UNSUPPORTED;
    }
    const bool rel = cfg->rel_buckets == 32;
    const int adapter0 = 5 + 16 * L + (has_head ? 4 : 0) + (rel ? 1 : 0);   // the adapter tensors come last
    const int pos0 = adapter0 + (A > 0 ? 4 * L : 0);                           // then DeBERTa's relative embeddings
    const int expect = pos0 + (PB > 0 ? 3 : 0);
    if (n_weights != expect) { set_error("rmu_encoder_create: expected " + std::to_string(expect) + " weight tensors"); return RMU_ERR_ARG; }
    if (rel && !w[adapter0 - 1]) { set_error("rmu_encoder_create: null relative attention bias"); return RMU_ERR_ARG; }
    for (int j = adapter0; j < pos0; ++j)
        if (!w[j]) { set_error("rmu_encoder_create: null adapter tensor"); return RMU_ERR_ARG; }
    for (int j = pos0; j < expect; ++j)
        if (!w[j]) { set_error("rmu_encoder_create: null relative embedding or LN_rel tensor"); return RMU_ERR_ARG; }
    if (H % 128 != 0 || F % 128 != 0 || H > 1024 || cfg->heads <= 0 || H % cfg->heads != 0 ||
        (H / cfg->heads != 32 && H / cfg->heads != 64)) {
        set_error("rmu_encoder_create: unsupported shape (hidden/ffn multiples of 128, hidden <= 1024, head_dim 32 or 64)");
        return RMU_ERR_UNSUPPORTED;
    }
    for (int l = 0; l < L; ++l) {
        static const char* const kName[] = {"query", "key", "value", "attention output", "intermediate", "output"};
        const int slot[] = {0, 2, 4, 6, 10, 12};                  // weight offsets within the layer's 16 tensors
        const size_t count[] = {size_t(H) * H, size_t(H) * H, size_t(H) * H, size_t(H) * H, size_t(F) * H, size_t(H) * F};
        for (int k = 0; k < 6; ++k) {
            const float* p = w[5 + 16 * l + slot[k]];
            if (!p) { set_error("rmu_encoder_create: null weight tensor"); return RMU_ERR_ARG; }
            const int rc = check_split_range("rmu_encoder_create", "layer " + std::to_string(l) + " " + kName[k], p, count[k]);
            if (rc != RMU_OK) return rc;
        }
    }
    for (int l = 0; l < L && A > 0; ++l) {
        for (int k = 0; k < 2; ++k) {                             // dense1 [A, H] and dense2 [H, A]
            const int rc = check_split_range("rmu_encoder_create",
                                             "layer " + std::to_string(l) + " adapter dense" + std::to_string(k + 1),
                                             w[adapter0 + 4 * l + 2 * k], static_cast<size_t>(A) * H);
            if (rc != RMU_OK) return rc;
        }
    }
    rmu_encoder* e = new_handle("rmu_encoder_create", *cfg, has_head);
    if (!e) return RMU_ERR_CUDA;
    e->ext = ext;
    e->qkv_w = 3 * H;
    e->ctx_w = H;
    e->has_x1 = e->has_cls_rows = true;
    int rc = RMU_OK;
    int i = 0;
    auto up = [&](float** dst, size_t n) { if (rc == RMU_OK) rc = upload(e, dst, w[i], n); ++i; };
    up(&e->word, static_cast<size_t>(cfg->vocab_size) * H);
    up(&e->pos, static_cast<size_t>(cfg->max_pos) * H);
    up(&e->typ, static_cast<size_t>(cfg->type_vocab) * H);
    up(&e->eg, H);
    up(&e->eb, H);
    e->layers.resize(L);
    for (int l = 0; l < L && rc == RMU_OK; ++l) {
        EncLayer& Ly = e->layers[l];
        const float *qw = w[i], *qb = w[i + 1], *kw = w[i + 2], *kb = w[i + 3], *vw = w[i + 4], *vb = w[i + 5];
        i += 6;
        rc = upload_split(e, &Ly.Wqkv, {qw, kw, vw}, H, H);
        if (rc == RMU_OK) {
            std::vector<float> bcat(3 * static_cast<size_t>(H));
            std::copy(qb, qb + H, bcat.begin());
            std::copy(kb, kb + H, bcat.begin() + H);
            std::copy(vb, vb + H, bcat.begin() + 2 * H);
            rc = upload(e, &Ly.bqkv, bcat.data(), bcat.size());
        }
        if (rc == RMU_OK) rc = upload_split(e, &Ly.Wo, {w[i]}, H, H);
        ++i;
        up(&Ly.bo, H);
        up(&Ly.ln1g, H);
        up(&Ly.ln1b, H);
        if (rc == RMU_OK) rc = upload_split(e, &Ly.W1, {w[i]}, F, H);
        ++i;
        up(&Ly.b1, F);
        if (rc == RMU_OK) rc = upload_split(e, &Ly.W2, {w[i]}, H, F);
        ++i;
        up(&Ly.b2, H);
        up(&Ly.ln2g, H);
        up(&Ly.ln2b, H);
    }
    if (rc == RMU_OK && L > 0) {
        const SplitOperand& W = e->layers[L - 1].Wqkv;
        const size_t kv = static_cast<size_t>(H) * H;
        rc = make_split_operand(&e->last_wq, W.hi, W.lo, H, H);
        if (rc == RMU_OK) rc = make_split_operand(&e->last_wkv, W.hi + kv, W.lo + kv, 2 * H, H);
    }
    if (has_head) {
        up(&e->pw, static_cast<size_t>(H) * H);
        up(&e->pb, H);
        up(&e->cw, static_cast<size_t>(cfg->num_labels) * H);
        up(&e->cb, cfg->num_labels);
    }
    if (rel && rc == RMU_OK) {
        std::vector<float> tab(static_cast<size_t>(cfg->heads) * kRelSpan);
        build_relative_bias_table(w[i], cfg->heads, tab.data());
        rc = upload(e, &e->rel, tab.data(), tab.size());
    }
    i = adapter0;
    for (int l = 0; l < L && A > 0 && rc == RMU_OK; ++l) {
        EncLayer& Ly = e->layers[l];
        rc = upload_split(e, &Ly.D1, {w[i]}, A, H);
        ++i;
        up(&Ly.d1, A);
        if (rc == RMU_OK) rc = upload_split(e, &Ly.D2, {w[i]}, H, A);
        ++i;
        up(&Ly.d2, H);
    }
    if (PB > 0 && rc == RMU_OK) {
        // R = LN_rel(rel_embeddings) once; per layer PQ' | PK = split((R [Wq; Wk]^T + [bq; bk]) * (col < H ? qscale : 1)),
        // the QKV epilogue's arithmetic on R, with q's scale log2(e) / sqrt(3 d_h)
        const int R2 = 2 * PB;
        float *rel_f = nullptr, *lng = nullptr, *lnb = nullptr;
        i = pos0;
        up(&rel_f, static_cast<size_t>(R2) * H);
        up(&lng, H);
        up(&lnb, H);
        SplitOperand Rp;
        __half *rh = nullptr, *rl = nullptr;
        if (rc == RMU_OK) rc = dev_alloc(e->allocs, &rh, static_cast<size_t>(R2) * H);
        if (rc == RMU_OK) rc = dev_alloc(e->allocs, &rl, static_cast<size_t>(R2) * H);
        if (rc == RMU_OK) rc = launch_layernorm(rel_f, R2, H, lng, lnb, cfg->ln_eps, rh, rl, nullptr);
        if (rc == RMU_OK) rc = make_split_operand(&Rp, rh, rl, R2, H);
        const float qs = 1.4426950408889634f / sqrtf(static_cast<float>(3 * (H / cfg->heads)));
        for (int l = 0; l < L && rc == RMU_OK; ++l) {
            EncLayer& Ly = e->layers[l];
            SplitOperand wqk;
            rc = make_split_operand(&wqk, Ly.Wqkv.hi, Ly.Wqkv.lo, 2 * H, H);
            if (rc == RMU_OK) rc = dev_alloc(e->allocs, &Ly.pos_hi, static_cast<size_t>(R2) * 2 * H);
            if (rc == RMU_OK) rc = dev_alloc(e->allocs, &Ly.pos_lo, static_cast<size_t>(R2) * 2 * H);
            if (rc != RMU_OK) break;
            GemmParams g{};
            g.M = R2; g.N = 2 * H; g.K = H; g.bias = Ly.bqkv; g.out_hi = Ly.pos_hi; g.out_lo = Ly.pos_lo; g.qcols = H; g.qscale = qs;
            rc = launch_gemm(GEMM_BIAS_SPLIT_QSCALE, Rp, wqk, g, e->sms, nullptr);
        }
        if (rc == RMU_OK) {
            const int rmax = cfg->max_pos - 1;
            e->cidx_h.resize(2 * static_cast<size_t>(rmax) + 1);
            build_position_index(PB, MRP, rmax, e->cidx_h.data());
            rc = dev_alloc(e->allocs, &e->cidx, e->cidx_h.size());
            if (rc == RMU_OK)
                RMU_CUDA(cudaMemcpy(e->cidx, e->cidx_h.data(), e->cidx_h.size() * sizeof(int), cudaMemcpyHostToDevice));
        }
        if (rc == RMU_OK) {
            const cudaError_t err = cudaDeviceSynchronize();
            if (err != cudaSuccess) { set_error(std::string("rmu_encoder_create: ") + cudaGetErrorString(err)); rc = RMU_ERR_CUDA; }
        }
    }
    if (rc != RMU_OK) { rmu_encoder_destroy(e); return rc; }
    *out = e;
    return RMU_OK;
}

// ModernBERT: GeGLU's Wi [2F, cols] (rows 0..F inputs, F..2F gates) -> 128-row blocks of 64 input rows followed by the
// 64 matching gate rows, so one E1 tile holds both halves of 64 output columns
static std::vector<float> geglu_rows(const float* w, int F, int cols) {
    std::vector<float> out(static_cast<size_t>(2) * F * cols);
    for (int k = 0; k < F / 64; ++k)
        for (int half = 0; half < 2; ++half)
            std::copy(w + (static_cast<size_t>(half) * F + 64 * k) * cols, w + (static_cast<size_t>(half) * F + 64 * k + 64) * cols,
                      out.begin() + (static_cast<size_t>(128) * k + 64 * half) * cols);
    return out;
}

int rmu_encoder_create_modernbert(const rmu_bert_config* cfg, const rmu_modernbert_ext* mb, const float* const* w,
                                  int n_weights, int has_head, rmu_encoder** out) {
    if (!cfg || !mb || !w || !out || !mb->half_window_h) { set_error("rmu_encoder_create_modernbert: bad argument"); return RMU_ERR_ARG; }
    const int H = cfg->hidden, F = cfg->ffn, L = cfg->layers, nh = cfg->heads;
    if (cfg->position_mode != RMU_POS_ABSOLUTE || cfg->rel_buckets != 0 || cfg->adapter_dim != 0) {
        set_error("rmu_encoder_create_modernbert: position_mode, rel_buckets and adapter_dim must be 0 (rotary positions, no "
                  "relative bias, no adapters)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (L < 1 || nh <= 0 || H % 128 != 0 || H > 1024 || H % nh != 0 || (H / nh != 32 && H / nh != 64) || F <= 0 ||
        F % 64 != 0 || cfg->vocab_size <= 0 || cfg->max_pos <= 0 || cfg->num_labels <= 0) {
        set_error("rmu_encoder_create_modernbert: unsupported shape (hidden a multiple of 128 up to 1024, head_dim 32 or 64, "
                  "intermediate_size a multiple of 64, at least one layer)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (mb->head_form != RMU_MB_HEAD_DENSE_GELU_LN) {
        set_error("rmu_encoder_create_modernbert: head_form must be RMU_MB_HEAD_DENSE_GELU_LN (0)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (mb->pooling != RMU_POOL_CLS && mb->pooling != RMU_POOL_MEAN) {
        set_error("rmu_encoder_create_modernbert: pooling must be RMU_POOL_CLS or RMU_POOL_MEAN");
        return RMU_ERR_ARG;
    }
    for (int l = 0; l < L; ++l)
        if (mb->half_window_h[l] < 0) {
            set_error("rmu_encoder_create_modernbert: layer " + std::to_string(l) + " has a negative half-window");
            return RMU_ERR_ARG;
        }
    const int DH = H / nh;
    if (mb->rope_rows != cfg->max_pos || mb->rope_half != DH / 2) {
        set_error("rmu_encoder_create_modernbert: the rope tables must be [max_pos, head_dim / 2] = [" +
                  std::to_string(cfg->max_pos) + ", " + std::to_string(DH / 2) + "]");
        return RMU_ERR_ARG;
    }
    const int head0 = 3 + 12 * L + 2, rope0 = head0 + (has_head ? 6 : 0), expect = rope0 + 4;
    if (n_weights != expect) {
        set_error("rmu_encoder_create_modernbert: expected " + std::to_string(expect) + " weight tensors");
        return RMU_ERR_ARG;
    }
    for (int j = 0; j < expect; ++j) {
        const bool layer0_attn_norm = j == 3 || j == 4;                // layer 0 has no attn_norm (identity)
        if (!w[j] && !layer0_attn_norm) {
            set_error(j >= rope0 ? "rmu_encoder_create_modernbert: null rope table"
                                 : "rmu_encoder_create_modernbert: null weight tensor " + std::to_string(j));
            return RMU_ERR_ARG;
        }
    }
    for (int l = 0; l < L; ++l) {
        static const char* const kName[] = {"Wqkv", "attention Wo", "mlp Wi", "mlp Wo"};
        const int slot[] = {2, 4, 8, 10};
        const size_t count[] = {size_t(3) * H * H, size_t(H) * H, size_t(2) * F * H, size_t(H) * F};
        for (int k = 0; k < 4; ++k) {
            // Wi as the checkpoint holds it, before geglu_rows reorders it
            const int rc = check_split_range("rmu_encoder_create_modernbert", "layer " + std::to_string(l) + " " + kName[k],
                                             w[3 + 12 * l + slot[k]], count[k]);
            if (rc != RMU_OK) return rc;
        }
    }
    rmu_encoder* e = new_handle("rmu_encoder_create_modernbert", *cfg, has_head);
    if (!e) return RMU_ERR_CUDA;
    e->modern = true;
    e->mb_pool = mb->pooling;
    e->qkv_w = 3 * H;
    e->ctx_w = H;
    e->has_x1 = e->has_cls_rows = e->has_posi = true;
    int rc = RMU_OK;
    int i = 0;
    auto up = [&](float** dst, size_t n) { if (rc == RMU_OK) rc = upload(e, dst, w[i], n); ++i; };
    up(&e->word, static_cast<size_t>(cfg->vocab_size) * H);
    up(&e->eg, H);
    up(&e->eb, H);
    const std::vector<float> zeros(H, 0.f);
    if (rc == RMU_OK) rc = upload(e, &e->pos, zeros.data(), H);
    if (rc == RMU_OK) rc = upload(e, &e->typ, zeros.data(), H);
    e->layers.resize(L);
    for (int l = 0; l < L && rc == RMU_OK; ++l) {
        EncLayer& Ly = e->layers[l];
        Ly.window = mb->half_window_h[l];
        if (l > 0) { up(&Ly.ln1g, H); up(&Ly.ln1b, H); } else i += 2;
        if (rc == RMU_OK) rc = upload_split(e, &Ly.Wqkv, {w[i]}, 3 * H, H);
        ++i;
        up(&Ly.bqkv, static_cast<size_t>(3) * H);
        if (rc == RMU_OK) rc = upload_split(e, &Ly.Wo, {w[i]}, H, H);
        ++i;
        up(&Ly.bo, H);
        up(&Ly.ln2g, H);
        up(&Ly.ln2b, H);
        if (rc == RMU_OK) {
            const std::vector<float> wi = geglu_rows(w[i], F, H);
            rc = upload_split(e, &Ly.W1, {wi.data()}, 2 * F, H);
        }
        ++i;
        if (rc == RMU_OK) {
            const std::vector<float> bi = geglu_rows(w[i], F, 1);
            rc = upload(e, &Ly.b1, bi.data(), bi.size());
        }
        ++i;
        if (rc == RMU_OK) rc = upload_split(e, &Ly.W2, {w[i]}, H, F);
        ++i;
        up(&Ly.b2, H);
    }
    up(&e->fng, H);
    up(&e->fnb, H);
    if (has_head) {
        up(&e->pw, static_cast<size_t>(H) * H);
        up(&e->pb, H);
        up(&e->hng, H);
        up(&e->hnb, H);
        up(&e->cw, static_cast<size_t>(cfg->num_labels) * H);
        up(&e->cb, cfg->num_labels);
    }
    const size_t tab = static_cast<size_t>(cfg->max_pos) * (DH / 2);
    up(&e->rope_cos[0], tab);
    up(&e->rope_sin[0], tab);
    up(&e->rope_cos[1], tab);
    up(&e->rope_sin[1], tab);
    if (rc != RMU_OK) { rmu_encoder_destroy(e); return rc; }
    *out = e;
    return RMU_OK;
}

}  // extern "C"

// the shape refusals of a decoder handle, before any CUDA call: hidden a multiple of 128 up to max_hidden (4096 on
// split planes, 8192 in NF4), head_dim 128, intermediate a multiple of 64, grouped kv heads, rope tables [max_pos, 64]
static int check_decoder_shape(const std::string& fn, const rmu_bert_config* cfg, const rmu_qwen3_ext* qx, int has_head,
                               int max_hidden) {
    const int H = cfg->hidden, F = cfg->ffn, L = cfg->layers, nh = cfg->heads, kv = qx->kv_heads;
    if (cfg->position_mode != RMU_POS_ABSOLUTE || cfg->rel_buckets != 0 || cfg->adapter_dim != 0) {
        set_error(fn + ": position_mode, rel_buckets and adapter_dim must be 0 (rotary positions, no "
                  "relative bias, no adapters)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (qx->head_dim != kQwenHD) {
        set_error(fn + ": head_dim must be 128, got " + std::to_string(qx->head_dim));
        return RMU_ERR_UNSUPPORTED;
    }
    if (H <= 0 || H % 128 != 0 || H > max_hidden) {
        set_error(fn + ": hidden_size must be a multiple of 128 up to " + std::to_string(max_hidden) + ", got " +
                  std::to_string(H));
        return RMU_ERR_UNSUPPORTED;
    }
    if (F <= 0 || F % 64 != 0) {
        set_error(fn + ": intermediate_size must be a positive multiple of 64, got " + std::to_string(F));
        return RMU_ERR_UNSUPPORTED;
    }
    if (nh <= 0 || kv <= 0 || nh % kv != 0) {
        set_error(fn + ": num_attention_heads must be a multiple of num_key_value_heads (" +
                  std::to_string(nh) + " heads, " + std::to_string(kv) + " kv heads)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (L < 1 || cfg->vocab_size <= 0 || cfg->max_pos <= 0 || cfg->num_labels <= 0) {
        set_error(fn + ": unsupported shape (at least one layer, positive vocab, max_pos, num_labels)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (qx->rope_rows != cfg->max_pos || qx->rope_half != kQwenHD / 2) {
        set_error(fn + ": the rope tables must be [max_pos, 64] = [" + std::to_string(cfg->max_pos) + ", 64]");
        return RMU_ERR_ARG;
    }
    if (qx->head_form != (has_head ? RMU_QWEN3_HEAD_LAST : RMU_QWEN3_HEAD_NONE)) {
        set_error(fn + ": head_form must be RMU_QWEN3_HEAD_LAST with a head, RMU_QWEN3_HEAD_NONE without");
        return RMU_ERR_ARG;
    }
    return RMU_OK;
}

// rmu_encoder_create_qwen3 (qk_norm) and rmu_encoder_create_llama (no q_norm / k_norm tensors: 9 per layer, no head);
// `who` prefixes the errors
static int create_decoder(const char* who, bool qk_norm, const rmu_bert_config* cfg, const rmu_qwen3_ext* qx,
                          const float* const* w, int n_weights, int has_head, rmu_encoder** out) {
    const std::string fn(who);
    if (!cfg || !qx || !w || !out) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    const int H = cfg->hidden, F = cfg->ffn, L = cfg->layers, nh = cfg->heads, kv = qx->kv_heads;
    const int shape_rc = check_decoder_shape(fn, cfg, qx, has_head, 4096);
    if (shape_rc != RMU_OK) return shape_rc;
    const int QD = nh * kQwenHD, KD = kv * kQwenHD, NQKV = QD + 2 * KD;
    const int per = qk_norm ? 11 : 9;                // tensors per layer
    const int norm0 = 1 + per * L, rope0 = norm0 + 1 + (has_head ? 1 : 0), expect = rope0 + 2;
    if (n_weights != expect) {
        set_error(fn + ": expected " + std::to_string(expect) + " weight tensors");
        return RMU_ERR_ARG;
    }
    for (int j = 0; j < expect; ++j)
        if (!w[j]) { set_error(fn + ": null weight tensor " + std::to_string(j)); return RMU_ERR_ARG; }
    for (int l = 0; l < L; ++l) {
        static const char* const kName[] = {"q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"};
        const int slot11[] = {1, 2, 3, 6, 8, 9, 10}, slot9[] = {1, 2, 3, 4, 6, 7, 8};
        const int* slot = qk_norm ? slot11 : slot9;
        const size_t count[] = {size_t(QD) * H, size_t(KD) * H, size_t(KD) * H, size_t(H) * QD, size_t(F) * H,
                                size_t(F) * H, size_t(H) * F};
        for (int k = 0; k < 7; ++k) {
            const int rc = check_split_range(fn, "layer " + std::to_string(l) + " " + kName[k], w[1 + per * l + slot[k]],
                                             count[k]);
            if (rc != RMU_OK) return rc;
        }
    }
    rmu_encoder* e = new_handle(fn, *cfg, has_head);
    if (!e) return RMU_ERR_CUDA;
    e->qwen = true;
    e->llama = !qk_norm;
    e->qext = *qx;
    e->qkv_w = NQKV;
    e->ctx_w = QD;
    e->has_qkvf = e->has_posi = true;
    int rc = RMU_OK;
    int i = 0;
    auto up = [&](float** dst, size_t n) { if (rc == RMU_OK) rc = upload(e, dst, w[i], n); ++i; };
    up(&e->word, static_cast<size_t>(cfg->vocab_size) * H);
    e->layers.resize(L);
    for (int l = 0; l < L && rc == RMU_OK; ++l) {
        EncLayer& Ly = e->layers[l];
        up(&Ly.ln1g, H);
        if (rc == RMU_OK) {
            std::vector<float> qkv(static_cast<size_t>(NQKV) * H);
            std::copy(w[i], w[i] + size_t(QD) * H, qkv.begin());
            std::copy(w[i + 1], w[i + 1] + size_t(KD) * H, qkv.begin() + size_t(QD) * H);
            std::copy(w[i + 2], w[i + 2] + size_t(KD) * H, qkv.begin() + size_t(QD + KD) * H);
            rc = upload_split(e, &Ly.Wqkv, {qkv.data()}, NQKV, H);
        }
        i += 3;
        if (qk_norm) {
            up(&Ly.qn, kQwenHD);
            up(&Ly.kn, kQwenHD);
        }
        if (rc == RMU_OK) rc = upload_split(e, &Ly.Wo, {w[i]}, H, QD);
        ++i;
        up(&Ly.ln2g, H);
        if (rc == RMU_OK) {
            // gate | up -> 128-row blocks of 64 gate rows (silu's input) and the 64 matching up rows
            std::vector<float> gu(static_cast<size_t>(2) * F * H);
            std::copy(w[i], w[i] + size_t(F) * H, gu.begin());
            std::copy(w[i + 1], w[i + 1] + size_t(F) * H, gu.begin() + size_t(F) * H);
            const std::vector<float> blocked = geglu_rows(gu.data(), F, H);
            rc = upload_split(e, &Ly.W1, {blocked.data()}, 2 * F, H);
        }
        i += 2;
        if (rc == RMU_OK) rc = upload_split(e, &Ly.W2, {w[i]}, H, F);
        ++i;
    }
    up(&e->fng, H);
    if (has_head) up(&e->cw, static_cast<size_t>(cfg->num_labels) * H);
    const size_t tab = static_cast<size_t>(cfg->max_pos) * (kQwenHD / 2);
    up(&e->rope_cos[0], tab);
    up(&e->rope_sin[0], tab);
    if (rc == RMU_OK) {
        const std::vector<float> zeros(static_cast<size_t>(std::max({NQKV, 2 * F, H})), 0.f);
        rc = upload(e, &e->zeros, zeros.data(), zeros.size());
    }
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->range_flag, 1);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->span_cu, 2);
    if (rc != RMU_OK) { rmu_encoder_destroy(e); return rc; }
    *out = e;
    return RMU_OK;
}

extern "C" {

int rmu_encoder_create_qwen3(const rmu_bert_config* cfg, const rmu_qwen3_ext* qx, const float* const* w, int n_weights,
                             int has_head, rmu_encoder** out) {
    return create_decoder("rmu_encoder_create_qwen3", true, cfg, qx, w, n_weights, has_head, out);
}

int rmu_encoder_create_llama(const rmu_bert_config* cfg, const rmu_qwen3_ext* qx, const float* const* w, int n_weights,
                             rmu_encoder** out) {
    if (qx && qx->head_form != RMU_QWEN3_HEAD_NONE) {
        set_error("rmu_encoder_create_llama: head_form must be RMU_QWEN3_HEAD_NONE (Llama runs without a head)");
        return RMU_ERR_ARG;
    }
    return create_decoder("rmu_encoder_create_llama", false, cfg, qx, w, n_weights, 0, out);
}

void rmu_encoder_destroy(rmu_encoder* e) {
    if (!e) return;
    cudaDeviceSynchronize();
    free_acts(e);
    for (DevBuf* b : {&e->span_ws, &e->dense_ws, &e->pos_ws, &e->d_ids, &e->d_typ, &e->d_cu, &e->d_out, &e->kv_cache, &e->gen_ws})
        b->release();
    for (void* p : e->allocs) cudaFree(p);
    if (e->ws_done) cudaEventDestroy(e->ws_done);
    delete e;
}

int rmu_encoder_embed(rmu_encoder* e, const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T,
                      int max_seqlen, int pool_mode, int normalize, float* out, void* stream) {
    int rc = check_batch(e, ids, cu, B, T, out);
    if (rc != RMU_OK) return rc;
    if (e->qwen) {
        if (pool_mode != RMU_POOL_LAST) { set_error("Qwen3 encoders pool by the last token only (RMU_POOL_LAST)"); return RMU_ERR_ARG; }
        std::lock_guard<std::mutex> g(e->mu);
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        rc = run_qwen3(e, ids, cu, B, T, max_seqlen, st);
        if (rc == RMU_OK) rc = qwen3_check_range(e, st);
        if (rc == RMU_OK)
            rc = launch_last_token(e->PRE, ids, cu, B, e->cfg.hidden, e->fng, e->cfg.ln_eps, -1, normalize, nullptr, 0, out, st);
        if (rc != RMU_OK) return rc;
        RMU_CUDA(cudaEventRecord(e->ws_done, st));
        return RMU_OK;
    }
    if (pool_mode != RMU_POOL_MEAN && pool_mode != RMU_POOL_CLS) { set_error("bad pool_mode"); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> g(e->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool cls = pool_mode == RMU_POOL_CLS && !e->modern;     // ModernBERT runs every layer in full
    rc = run_encoder(e, ids, type_ids, cu, B, T, max_seqlen, cls, st);
    if (rc != RMU_OK) return rc;
    const SplitOperand& h = cls ? e->X_cls : e->X;
    if (e->dense_w.empty())
        rc = launch_pool(h.hi, h.lo, cu, B, e->cfg.hidden, pool_mode, normalize, cls, out, st);
    else
        rc = run_dense(e, h, cu, B, pool_mode, cls, normalize, out, st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

int rmu_encoder_classify(rmu_encoder* e, const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T,
                         int max_seqlen, float* out, void* stream) {
    int rc = check_batch(e, ids, cu, B, T, out);
    if (rc != RMU_OK) return rc;
    if (!e->has_head) { set_error("rmu_encoder_classify: encoder was created without a classification head"); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> g(e->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (e->qwen) {
        rc = run_qwen3(e, ids, cu, B, T, max_seqlen, st);
        if (rc == RMU_OK) rc = qwen3_check_range(e, st);
        if (rc == RMU_OK)
            rc = launch_last_token(e->PRE, ids, cu, B, e->cfg.hidden, e->fng, e->cfg.ln_eps, e->qext.pad_token_id, 0, e->cw,
                                   e->cfg.num_labels, out, st);
        if (rc != RMU_OK) return rc;
        RMU_CUDA(cudaEventRecord(e->ws_done, st));
        return RMU_OK;
    }
    rc = run_encoder(e, ids, type_ids, cu, B, T, max_seqlen, true, st);
    if (rc != RMU_OK) return rc;
    if (e->modern) {
        // pool the final hidden state (CLS or mean) into PRE_cls, then the head
        rc = launch_pool(e->X.hi, e->X.lo, cu, B, e->cfg.hidden, e->mb_pool, 0, false, e->PRE_cls, st);
        if (rc == RMU_OK)
            rc = launch_mb_head(e->PRE_cls, B, e->cfg.hidden, e->cfg.num_labels, e->pw, e->pb, e->hng, e->hnb, e->cfg.ln_eps,
                                e->cw, e->cb, out, st);
        if (rc != RMU_OK) return rc;
        RMU_CUDA(cudaEventRecord(e->ws_done, st));
        return RMU_OK;
    }
    rc = launch_cls_head(e->X_cls.hi, e->X_cls.lo, cu, B, e->cfg.hidden, e->cfg.num_labels, true, e->pw, e->pb, e->cw, e->cb,
                         out, st, e->ext.head_act);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

int rmu_encoder_hidden(rmu_encoder* e, const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T,
                       int max_seqlen, float* out, void* stream) {
    int rc = check_batch(e, ids, cu, B, T, out);
    if (rc != RMU_OK) return rc;
    std::lock_guard<std::mutex> g(e->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (e->qwen) {
        // the final norm into the X planes, then joined like every other encoder's hidden state
        rc = run_qwen3(e, ids, cu, B, T, max_seqlen, st);
        if (rc == RMU_OK) rc = launch_rms_split(e->PRE, T, e->cfg.hidden, e->fng, e->cfg.ln_eps, e->X.hi, e->X.lo, e->range_flag, st);
        if (rc == RMU_OK) rc = qwen3_check_range(e, st);
    } else {
        rc = run_encoder(e, ids, type_ids, cu, B, T, max_seqlen, false, st);
    }
    if (rc != RMU_OK) return rc;
    rc = launch_join_planes(e->X.hi, e->X.lo, static_cast<size_t>(T) * e->cfg.hidden, out, st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

int rmu_decoder_attention_spans(rmu_encoder* e, const int32_t* ids, int T, const int32_t* spans, int n_spans, double* out,
                                void* stream) {
    const std::string fn("rmu_decoder_attention_spans");
    if (!e || !ids || !spans || !out || T <= 0 || n_spans <= 0) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    int rc = check_decoder(e, fn);
    if (rc == RMU_OK) rc = check_nf4_intact(e, fn);
    if (rc != RMU_OK) return rc;
    if (T > e->cfg.max_pos) {
        set_error(fn + ": " + std::to_string(T) + " tokens exceed max_position_embeddings (" + std::to_string(e->cfg.max_pos) +
                  ")");
        return RMU_ERR_ARG;
    }
    std::lock_guard<std::mutex> g(e->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int cu_h[2] = {0, T};
    // pageable source: the copy has taken cu_h when the call returns; span_cu is read by run_qwen3 only, which the
    // range check below has finished before this entry point returns
    RMU_CUDA(cudaMemcpyAsync(e->span_cu, cu_h, sizeof(cu_h), cudaMemcpyHostToDevice, st));
    rc = run_qwen3(e, ids, e->span_cu, 1, T, T, st, true);
    if (rc == RMU_OK) rc = qwen3_check_range(e, st);
    if (rc == RMU_OK) rc = grow(e->span_ws, attention_spans_ws_floats(T, e->cfg.heads) * sizeof(float));
    if (rc == RMU_OK)
        rc = launch_attention_spans(e->QKVP.hi, e->QKVP.lo, T, e->cfg.heads, e->qext.kv_heads, spans, n_spans,
                                    e->span_ws.as<float>(), out, st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

// host_mu held: the staging buffers belong to the *_host entry points only
static int stage_batch(rmu_encoder* e, const int32_t* ids_h, const int32_t* typ_h, const int32_t* cu_h, int B, int T,
                       cudaStream_t st) {
    const size_t i4 = sizeof(int32_t), out_w = std::max(embed_width(e), e->cfg.num_labels);
    int rc = grow(e->d_ids, T * i4, token_rows(T) * i4);
    if (rc == RMU_OK) rc = grow(e->d_typ, T * i4, token_rows(T) * i4);
    if (rc == RMU_OK) rc = grow(e->d_cu, (B + 1) * i4, seq_rows(B) * i4);
    if (rc == RMU_OK) rc = grow(e->d_out, B * out_w * sizeof(float), seq_rows(B) * out_w * sizeof(float));
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(e->d_ids.p, ids_h, T * i4, cudaMemcpyHostToDevice, st));
    if (typ_h) RMU_CUDA(cudaMemcpyAsync(e->d_typ.p, typ_h, T * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(e->d_cu.p, cu_h, (B + 1) * i4, cudaMemcpyHostToDevice, st));
    return RMU_OK;
}

int rmu_encoder_embed_host(rmu_encoder* e, const int32_t* ids_h, const int32_t* typ_h, const int32_t* cu_h, int B, int T,
                           int max_seqlen, int pool_mode, int normalize, float* out_h, void* stream) {
    int rc = check_batch(e, ids_h, cu_h, B, T, out_h);
    if (rc != RMU_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::lock_guard<std::mutex> hg(e->host_mu);
    rc = stage_batch(e, ids_h, typ_h, cu_h, B, T, st);
    if (rc != RMU_OK) return rc;
    rc = rmu_encoder_embed(e, e->d_ids.as<int32_t>(), typ_h ? e->d_typ.as<int32_t>() : nullptr, e->d_cu.as<int32_t>(), B, T,
                           max_seqlen, pool_mode, normalize, e->d_out.as<float>(), st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(out_h, e->d_out.p, static_cast<size_t>(B) * embed_width(e) * sizeof(float), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    return RMU_OK;
}

int rmu_encoder_classify_host(rmu_encoder* e, const int32_t* ids_h, const int32_t* typ_h, const int32_t* cu_h, int B,
                              int T, int max_seqlen, float* out_h, void* stream) {
    int rc = check_batch(e, ids_h, cu_h, B, T, out_h);
    if (rc != RMU_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::lock_guard<std::mutex> hg(e->host_mu);
    rc = stage_batch(e, ids_h, typ_h, cu_h, B, T, st);
    if (rc != RMU_OK) return rc;
    rc = rmu_encoder_classify(e, e->d_ids.as<int32_t>(), typ_h ? e->d_typ.as<int32_t>() : nullptr, e->d_cu.as<int32_t>(), B, T,
                              max_seqlen, e->d_out.as<float>(), st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(out_h, e->d_out.p, static_cast<size_t>(B) * e->cfg.num_labels * sizeof(float), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    return RMU_OK;
}

int rmu_encoder_set_dense(rmu_encoder* e, int n_layers, const int32_t* dims, const float* const* W_h, const float* const* b_h,
                          const int32_t* acts) {
    if (!e || n_layers <= 0 || !dims || !W_h || !acts) { set_error("rmu_encoder_set_dense: bad argument"); return RMU_ERR_ARG; }
    if (e->qwen) {
        set_error("rmu_encoder_set_dense: Qwen3 and Llama encoders take no Dense modules (their last-token kernel "
                  "normalises its row itself)");
        return RMU_ERR_UNSUPPORTED;
    }
    if (dims[0] != e->cfg.hidden) {
        set_error("rmu_encoder_set_dense: dims[0] = " + std::to_string(dims[0]) + " must equal hidden (" +
                  std::to_string(e->cfg.hidden) + ")");
        return RMU_ERR_ARG;
    }
    for (int l = 0; l < n_layers; ++l) {
        if (dims[l + 1] <= 0 || !W_h[l]) {
            set_error("rmu_encoder_set_dense: layer " + std::to_string(l) + " needs a positive width and a weight");
            return RMU_ERR_ARG;
        }
        if (acts[l] != RMU_DENSE_IDENTITY && acts[l] != RMU_DENSE_TANH) {
            set_error("rmu_encoder_set_dense: act must be RMU_DENSE_IDENTITY (0) or RMU_DENSE_TANH (1)");
            return RMU_ERR_UNSUPPORTED;
        }
    }
    std::lock_guard<std::mutex> hg(e->host_mu);
    std::lock_guard<std::mutex> g(e->mu);
    if (!e->dense_w.empty()) { set_error("rmu_encoder_set_dense: a projection is already attached"); return RMU_ERR_ARG; }
    std::vector<float*> w(n_layers, nullptr), b(n_layers, nullptr);
    for (int l = 0; l < n_layers; ++l) {
        int rc = upload(e, &w[l], W_h[l], static_cast<size_t>(dims[l + 1]) * dims[l]);
        if (rc == RMU_OK && b_h && b_h[l]) rc = upload(e, &b[l], b_h[l], dims[l + 1]);
        if (rc != RMU_OK) return rc;
    }
    e->dense_dims.assign(dims, dims + n_layers + 1);
    e->dense_w = w;
    e->dense_b = b;
    e->dense_act.assign(acts, acts + n_layers);
    return RMU_OK;
}

int rmu_decoder_set_lm_head(rmu_encoder* e, const float* W_h) {
    if (!e || !W_h) { set_error("rmu_decoder_set_lm_head: bad argument"); return RMU_ERR_ARG; }
    int rc = check_decoder(e, "rmu_decoder_set_lm_head");
    if (rc != RMU_OK) return rc;
    const int V = e->cfg.vocab_size, H = e->cfg.hidden;
    if (V % 128 != 0) {
        set_error("rmu_decoder_set_lm_head: vocab_size must be a multiple of 128 (the LM head GEMM's tile), got " +
                  std::to_string(V));
        return RMU_ERR_UNSUPPORTED;
    }
    std::lock_guard<std::mutex> hg(e->host_mu);
    std::lock_guard<std::mutex> g(e->mu);
    if (e->has_lm_head) { set_error("rmu_decoder_set_lm_head: an LM head is already attached"); return RMU_ERR_ARG; }
    rc = check_split_range("rmu_decoder_set_lm_head", "lm_head", W_h, static_cast<size_t>(V) * H);
    if (rc != RMU_OK) return rc;
    rc = upload_split(e, &e->lm_head, {W_h}, V, H);
    if (rc == RMU_OK) {
        const std::vector<float> zeros(static_cast<size_t>(V), 0.f);
        rc = upload(e, &e->lm_zero, zeros.data(), zeros.size());
    }
    if (rc != RMU_OK) return rc;
    e->has_lm_head = true;
    return RMU_OK;
}

int rmu_decoder_quantize_nf4(rmu_encoder* e, void* stream) {
    const std::string fn("rmu_decoder_quantize_nf4");
    if (!e) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    int rc = check_decoder(e, fn);
    if (rc != RMU_OK) return rc;
    const rmu_bert_config& c = e->cfg;
    const int H = c.hidden, F = c.ffn, QD = c.heads * kQwenHD, NQKV = e->qkv_w;
    // K of q | k | v, o, gate | up, down.  K % 64 == 0 keeps every quantisation block inside one row, so the handle's
    // row orders (the fused q | k | v rows, W1's 64 + 64 gate / up blocks) move whole blocks and give the codes of the
    // checkpoint's own tensors.
    const int64_t shape[4][2] = {{NQKV, H}, {H, QD}, {2 * static_cast<int64_t>(F), H}, {H, F}};
    for (const auto& sh : shape) {
        if (sh[1] % kNf4Block != 0 || sh[1] > kNf4MaxK) {
            set_error(fn + ": every projection's K must be a multiple of 64 up to " + std::to_string(kNf4MaxK) + ", got " +
                      std::to_string(sh[1]));
            return RMU_ERR_UNSUPPORTED;
        }
    }
    std::lock_guard<std::mutex> hg(e->host_mu);
    std::lock_guard<std::mutex> g(e->mu);
    if (e->nf4 || e->nf4_broken) { set_error(fn + ": the handle's weights are already NF4"); return RMU_ERR_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RMU_CUDA(cudaDeviceSynchronize());                 // work queued on any stream may still read the split planes
    int64_t delta = 0, peak = 0;
    auto release = [&](void* p, int64_t bytes) -> int {
        e->allocs.erase(std::find(e->allocs.begin(), e->allocs.end(), p));
        RMU_CUDA(cudaFree(p));
        delta -= bytes;
        return RMU_OK;
    };
    auto convert = [&](EncLayer& L, int w) -> int {
        SplitOperand& S = L.*kDecoderSplit[w];
        Nf4Weight& Q = L.nf4[w];
        const int64_t n = shape[w][0] * shape[w][1];
        // the quantiser reads hi only: lo goes first, so the codes never raise the handle above its starting bytes.
        // S is cleared at once: no tensor map over a freed plane outlives this call, even if it fails below.
        __half* hi = S.hi;
        void* lo = S.lo;
        S = SplitOperand{};
        int rc = release(lo, n * 2);
        if (rc == RMU_OK) rc = dev_alloc(e->allocs, &Q.codes, n / 2);
        if (rc == RMU_OK) rc = dev_alloc(e->allocs, &Q.absmax, n / kNf4Block);
        if (rc != RMU_OK) return rc;
        delta += n / 2 + n / kNf4Block * 4;
        peak = std::max(peak, delta);
        Q.rows = static_cast<int>(shape[w][0]);
        Q.cols = static_cast<int>(shape[w][1]);
        rc = launch_nf4_quantize(hi, n, Q.codes, Q.absmax, st);
        if (rc != RMU_OK) return rc;
        RMU_CUDA(cudaStreamSynchronize(st));
        return release(hi, n * 2);
    };
    e->nf4_broken = true;                              // until every layer is converted
    for (int l = 0; l < c.layers && rc == RMU_OK; ++l)
        for (int w = 0; w < 4 && rc == RMU_OK; ++w) rc = convert(e->layers[l], w);
    // the prefill's scratch, allocated once the split planes are gone: one hi | lo pair as large as the largest weight
    int64_t most = 0;
    for (const auto& sh : shape) most = std::max(most, sh[0] * sh[1]);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->nf4_hi, most);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->nf4_lo, most);
    if (rc != RMU_OK) return rc;
    delta += most * 4;
    peak = std::max(peak, delta);
    RMU_CUDA(cudaMemset(e->nf4_lo, 0, most * sizeof(__half)));
    for (int w = 0; w < 4 && rc == RMU_OK; ++w)
        rc = make_split_operand(&e->nf4_op[w], e->nf4_hi, e->nf4_lo, shape[w][0], static_cast<int>(shape[w][1]));
    if (rc != RMU_OK) return rc;
    e->nf4 = true;
    e->nf4_broken = false;
    e->nf4_peak = peak;
    e->nf4_delta = delta;
    return RMU_OK;
}

// the [rows, cols] shapes of a decoder layer's four projections (q | k | v, o, gate | up, down) in the handle's row order
static void decoder_shapes(const rmu_encoder* e, int64_t shape[4][2]) {
    const int64_t H = e->cfg.hidden, F = e->cfg.ffn, QD = static_cast<int64_t>(e->cfg.heads) * kQwenHD;
    const int64_t s[4][2] = {{e->qkv_w, H}, {H, QD}, {2 * F, H}, {H, F}};
    std::memcpy(shape, s, sizeof(s));
}

int rmu_decoder_create_nf4(const rmu_bert_config* cfg, const rmu_qwen3_ext* qx, int qk_norm, const float* embed_h,
                           const float* final_norm_h, const float* rope_cos_h, const float* rope_sin_h,
                           rmu_encoder** out) {
    const std::string fn("rmu_decoder_create_nf4");
    if (!cfg || !qx || !embed_h || !final_norm_h || !rope_cos_h || !rope_sin_h || !out || (qk_norm != 0 && qk_norm != 1)) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    int rc = check_decoder_shape(fn, cfg, qx, 0, kRmsMaxHidden);
    if (rc != RMU_OK) return rc;
    const int H = cfg->hidden, F = cfg->ffn, QD = cfg->heads * kQwenHD, NQKV = QD + 2 * qx->kv_heads * kQwenHD;
    const int64_t K[4] = {H, QD, H, F};
    for (int64_t k : K) {
        if (k % kNf4Block != 0 || k > kNf4MaxK) {
            set_error(fn + ": every projection's K must be a multiple of 64 up to " + std::to_string(kNf4MaxK) + ", got " +
                      std::to_string(k));
            return RMU_ERR_UNSUPPORTED;
        }
    }
    rmu_encoder* e = new_handle(fn, *cfg, 0);
    if (!e) return RMU_ERR_CUDA;
    e->qwen = true;
    e->llama = !qk_norm;
    e->qext = *qx;
    e->qkv_w = NQKV;
    e->ctx_w = QD;
    e->has_qkvf = e->has_posi = true;
    e->nf4 = e->by_layer = true;
    e->layers.resize(cfg->layers);
    const size_t tab = static_cast<size_t>(cfg->max_pos) * (kQwenHD / 2);
    rc = upload(e, &e->word, embed_h, static_cast<size_t>(cfg->vocab_size) * H);
    if (rc == RMU_OK) rc = upload(e, &e->fng, final_norm_h, H);
    if (rc == RMU_OK) rc = upload(e, &e->rope_cos[0], rope_cos_h, tab);
    if (rc == RMU_OK) rc = upload(e, &e->rope_sin[0], rope_sin_h, tab);
    if (rc == RMU_OK) {
        const std::vector<float> zeros(static_cast<size_t>(std::max({NQKV, 2 * F, H})), 0.f);
        rc = upload(e, &e->zeros, zeros.data(), zeros.size());
    }
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->range_flag, 1);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->span_cu, 2);
    // the prefill's scratch hi | lo pair (lo all zero), the size of the largest projection; each layer's load also
    // builds its projections' hi planes in it
    int64_t shape[4][2];
    decoder_shapes(e, shape);
    int64_t most = 0;
    for (const auto& sh : shape) most = std::max(most, sh[0] * sh[1]);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->nf4_hi, most);
    if (rc == RMU_OK) rc = dev_alloc(e->allocs, &e->nf4_lo, most);
    if (rc == RMU_OK && cudaMemset(e->nf4_lo, 0, most * sizeof(__half)) != cudaSuccess) {
        set_error(fn + ": " + cudaGetErrorString(cudaGetLastError()));
        rc = RMU_ERR_CUDA;
    }
    for (int w = 0; w < 4 && rc == RMU_OK; ++w)
        rc = make_split_operand(&e->nf4_op[w], e->nf4_hi, e->nf4_lo, shape[w][0], static_cast<int>(shape[w][1]));
    if (rc != RMU_OK) { rmu_encoder_destroy(e); return rc; }
    *out = e;
    return RMU_OK;
}

// fp32 elements of one staging chunk of rmu_decoder_load_layer_nf4 (64 MiB, plus 32 MiB for the lo plane the split
// kernel also writes, which the quantiser never reads)
constexpr size_t kNf4LoadChunk = size_t(1) << 24;

int rmu_decoder_load_layer_nf4(rmu_encoder* e, int layer, const float* const* w, void* stream) {
    const std::string fn("rmu_decoder_load_layer_nf4");
    if (!e || !w) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    int rc = check_decoder(e, fn);
    if (rc != RMU_OK) return rc;
    if (!e->by_layer) { set_error(fn + ": the handle must come from rmu_decoder_create_nf4"); return RMU_ERR_ARG; }
    const rmu_bert_config& c = e->cfg;
    if (layer < 0 || layer >= c.layers) {
        set_error(fn + ": layer " + std::to_string(layer) + " is outside the model's " + std::to_string(c.layers) +
                  " layers");
        return RMU_ERR_ARG;
    }
    const bool qk = !e->llama;
    const int per = qk ? 11 : 9;
    for (int j = 0; j < per; ++j)
        if (!w[j]) { set_error(fn + ": layer " + std::to_string(layer) + ": null weight tensor " + std::to_string(j)); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> hg(e->host_mu);
    std::lock_guard<std::mutex> g(e->mu);
    if (layer != e->layers_loaded) {
        set_error(fn + ": layers load in order: expected layer " + std::to_string(e->layers_loaded) + " of " +
                  std::to_string(c.layers) + ", got " + std::to_string(layer));
        return RMU_ERR_ARG;
    }
    const int H = c.hidden, F = c.ffn, QD = c.heads * kQwenHD, KD = e->qext.kv_heads * kQwenHD;
    static const char* const kName[] = {"q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"};
    const int slot11[] = {1, 2, 3, 6, 8, 9, 10}, slot9[] = {1, 2, 3, 4, 6, 7, 8};
    const int* slot = qk ? slot11 : slot9;
    const size_t count[] = {size_t(QD) * H, size_t(KD) * H, size_t(KD) * H, size_t(H) * QD, size_t(F) * H,
                            size_t(F) * H, size_t(H) * F};
    for (int k = 0; k < 7; ++k) {
        rc = check_split_range(fn, "layer " + std::to_string(layer) + " " + kName[k], w[slot[k]], count[k]);
        if (rc != RMU_OK) return rc;
    }
    const float *q = w[slot[0]], *kw = w[slot[1]], *v = w[slot[2]], *o = w[slot[3]];
    const float *gate = w[slot[4]], *up = w[slot[5]], *down = w[slot[6]];
    // each projection as runs of consecutive source elements in the handle's row order: q | k | v; o; gate | up in
    // 128-row blocks of 64 gate rows and the 64 matching up rows (geglu_rows); down
    std::vector<std::pair<const float*, size_t>> runs[4];
    runs[0] = {{q, count[0]}, {kw, count[1]}, {v, count[2]}};
    runs[1] = {{o, count[3]}};
    for (int b = 0; b < F / 64; ++b) {
        runs[2].push_back({gate + size_t(64) * b * H, size_t(64) * H});
        runs[2].push_back({up + size_t(64) * b * H, size_t(64) * H});
    }
    runs[3] = {{down, count[6]}};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    EncLayer& Ly = e->layers[layer];
    // a retry after a failed load reuses what the failed attempt allocated
    auto vec = [&](float** dst, const float* src, size_t n) -> int {
        if (!*dst) {
            const int r = dev_alloc(e->allocs, dst, n);
            if (r != RMU_OK) return r;
        }
        RMU_CUDA(cudaMemcpy(*dst, src, n * sizeof(float), cudaMemcpyHostToDevice));
        return RMU_OK;
    };
    rc = vec(&Ly.ln1g, w[0], H);
    if (rc == RMU_OK) rc = vec(&Ly.ln2g, w[qk ? 7 : 5], H);
    if (rc == RMU_OK && qk) rc = vec(&Ly.qn, w[4], kQwenHD);
    if (rc == RMU_OK && qk) rc = vec(&Ly.kn, w[5], kQwenHD);
    if (rc != RMU_OK) return rc;
    int64_t shape[4][2];
    decoder_shapes(e, shape);
    void* stage = nullptr;
    RMU_CUDA(cudaMalloc(&stage, kNf4LoadChunk * (sizeof(float) + sizeof(__half))));
    float* stage_f = static_cast<float*>(stage);
    __half* stage_lo = reinterpret_cast<__half*>(stage_f + kNf4LoadChunk);
    // the same hi plane as upload_split's launch_split_planes, built chunk by chunk in the prefill scratch, then the
    // same quantiser as rmu_decoder_quantize_nf4: the same codes and absmax
    for (int p = 0; p < 4 && rc == RMU_OK; ++p) {
        Nf4Weight& Q = Ly.nf4[p];
        const int64_t n = shape[p][0] * shape[p][1];
        if (!Q.codes) rc = dev_alloc(e->allocs, &Q.codes, n / 2);
        if (rc == RMU_OK && !Q.absmax) rc = dev_alloc(e->allocs, &Q.absmax, n / kNf4Block);
        if (rc != RMU_OK) break;
        Q.rows = static_cast<int>(shape[p][0]);
        Q.cols = static_cast<int>(shape[p][1]);
        size_t done = 0, fill = 0;
        auto flush = [&]() -> int {
            const int r = launch_split_planes(stage_f, fill, e->nf4_hi + done, stage_lo, st);
            done += fill;
            fill = 0;
            return r;
        };
        for (const auto& run : runs[p]) {
            for (size_t at = 0; at < run.second && rc == RMU_OK;) {
                const size_t take = std::min(run.second - at, kNf4LoadChunk - fill);
                if (cudaMemcpyAsync(stage_f + fill, run.first + at, take * sizeof(float), cudaMemcpyHostToDevice, st) !=
                    cudaSuccess) {
                    set_error(fn + ": " + cudaGetErrorString(cudaGetLastError()));
                    rc = RMU_ERR_CUDA;
                    break;
                }
                fill += take;
                at += take;
                if (fill == kNf4LoadChunk) rc = flush();
            }
            if (rc != RMU_OK) break;
        }
        if (rc == RMU_OK) rc = flush();
        if (rc == RMU_OK) rc = launch_nf4_quantize(e->nf4_hi, n, Q.codes, Q.absmax, st);
    }
    const cudaError_t err = cudaStreamSynchronize(st);
    cudaFree(stage);
    if (rc != RMU_OK) return rc;
    if (err != cudaSuccess) { set_error(fn + ": " + cudaGetErrorString(err)); return RMU_ERR_CUDA; }
    e->layers_loaded = layer + 1;
    return RMU_OK;
}

int rmu_decoder_generate(rmu_encoder* e, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                         int max_new_tokens, int32_t* out_h, int32_t* n_out, float* logits_h, void* stream) {
    const std::string fn("rmu_decoder_generate");
    if (!e || !ids_h || !s || !out_h || !n_out || T < 1 || max_new_tokens < 1) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    const int rc = check_generate(e, fn, ids_h, T, s);
    if (rc != RMU_OK) return rc;
    std::scoped_lock lk(e->host_mu, e->mu);
    return generate_loop(e, fn, ids_h, T, s, seed, max_new_tokens, 0, Drafter(), out_h, n_out, logits_h, nullptr, stream);
}

int rmu_prompt_lookup_draft(const int32_t* ids, int n, int k, int max_ngram, int max_len, int32_t* out) {
    if (!ids || !out || n < 1 || k < 1 || max_ngram < 1) { set_error("rmu_prompt_lookup_draft: bad argument"); return RMU_ERR_ARG; }
    if (max_len == n + 1) return 0;                      // the model's own next token already reaches max_len
    for (int g = std::min(max_ngram, n - 1); g > 0; --g) {
        const int32_t* tail = ids + n - g;
        for (int i = 0; i + g <= n; ++i) {
            if (!std::equal(ids + i, ids + i + g, tail)) continue;
            const int start = i + g, end = std::min({start + k, n, max_len});
            if (start < end) {
                std::copy(ids + start, ids + end, out);
                return end - start;
            }
        }
    }
    return 0;
}

int rmu_decoder_generate_lookup(rmu_encoder* e, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                                int max_new_tokens, int lookup_tokens, int max_ngram, int32_t* out_h, int32_t* n_out,
                                float* logits_h, int32_t* n_passes, void* stream) {
    const std::string fn("rmu_decoder_generate_lookup");
    if (!e || !ids_h || !s || !out_h || !n_out || T < 1 || max_new_tokens < 1 || lookup_tokens < 0 || max_ngram < 1) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    const int rc = check_generate(e, fn, ids_h, T, s);
    if (rc != RMU_OK) return rc;
    std::scoped_lock lk(e->host_mu, e->mu);
    const int max_len = T + max_new_tokens;              // transformers' max_length
    const Drafter draft = [&](const std::vector<int32_t>& seq, int k, int32_t* out) {
        return std::max(0, rmu_prompt_lookup_draft(seq.data(), static_cast<int>(seq.size()), k, max_ngram, max_len, out));
    };
    return generate_loop(e, fn, ids_h, T, s, seed, max_new_tokens, std::min(lookup_tokens, kMaxDrafts), draft, out_h,
                         n_out, logits_h, n_passes, stream);
}

int rmu_debug_generate_drafts(rmu_encoder* e, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                              int max_new_tokens, const int32_t* drafts_h, int k, int32_t* out_h, int32_t* n_out,
                              float* logits_h, int32_t* n_passes, void* stream) {
    const std::string fn("rmu_debug_generate_drafts");
    if (!e || !ids_h || !s || !drafts_h || !out_h || !n_out || T < 1 || max_new_tokens < 1 || k < 0) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    if (check_decoder(e, fn) != RMU_OK) return RMU_ERR_ARG;
    for (int i = 0; i < max_new_tokens; ++i)
        if (drafts_h[i] < 0 || drafts_h[i] >= e->cfg.vocab_size) { set_error(fn + ": draft id out of range"); return RMU_ERR_ARG; }
    const int rc = check_generate(e, fn, ids_h, T, s);
    if (rc != RMU_OK) return rc;
    std::scoped_lock lk(e->host_mu, e->mu);
    // the draft at output index n: drafts_h[n .. n + k)
    const Drafter draft = [&](const std::vector<int32_t>& seq, int kk, int32_t* out) {
        std::copy(drafts_h + (seq.size() - T), drafts_h + (seq.size() - T) + kk, out);
        return kk;
    };
    return generate_loop(e, fn, ids_h, T, s, seed, max_new_tokens, std::min(k, kMaxDrafts), draft, out_h, n_out, logits_h,
                         n_passes, stream);
}

// The draft-model drafter of rmu_decoder_generate_assisted (DESIGN.md, "Speculative decoding with a draft model").  It
// keeps dvalid, the leading positions of seq whose k / v the draft's cache holds for the right tokens.  A call with
// the pending token at p = |seq| - 1 (output index n = |seq| - T) runs, on the draft handle: the prompt's prefill the
// first time (dvalid = T); catch-up rows dvalid .. p through run_decode_rows, in runs of at most kRun rows, the last
// row's logits giving draft 1; then k - 1 single-row steps, step j feeding draft j - 1, whose id the previous sampler
// wrote on the device.  Draft j samples with the target's settings, presence bits seq + drafts 1 .. j - 1 (the sampler
// sets each chosen bit) and Philox(seed, n + j - 1): as the target's verify row j - 1 samples.  One synchronise at the
// end reads the drafts and the draft's range flag; a raised flag is cleared and the pass gets no drafts.  The next
// call sets dvalid from how many drafts seq kept, and the heuristic schedule moves k from whether all of them were.
struct ModelDrafter {
    static constexpr int kRun = kMaxDrafts + 1;           // catch-up rows per run_decode_rows
    rmu_encoder* d;
    cudaStream_t st;
    const int32_t* ids_h;
    int T, dcap, schedule, kcur;
    SampleArgs sa;
    uint64_t seed;
    float *logits = nullptr, *part = nullptr;            // the draft's gen_ws: logits [V] | presence [words] | drafts
    unsigned* presence = nullptr;                          // [kMaxDrafts] | decode partials [kRun rows] | ints: ids
    int *tok = nullptr, *ints = nullptr;                   // [kRun] | shift [kRun] (zeros)
    size_t words;
    std::vector<unsigned> bits;                            // seq[0 .. folded)'s presence bits
    size_t folded = 0;
    std::vector<int32_t> last;                             // the drafts the last call proposed, at last_p + 1 ..
    int last_p = -1, dvalid = 0;
    bool prefilled = false;

    size_t layout(void* base) {
        Carve w(base);
        logits = w.take<float>(d->cfg.vocab_size);
        presence = w.take<unsigned>(words);
        tok = w.take<int>(kMaxDrafts);
        part = w.take<float>(kRun * decode_part_floats(d->cfg.heads, dcap));
        ints = w.take<int>(2 * kRun);
        return w.size;
    }

    // the draft's cache, workspace and staging for this call; then st waits for the draft's last use
    int setup(const std::string& fn) {
        words = (static_cast<size_t>(d->cfg.vocab_size) + 31) / 32;
        bits.assign(words, 0u);
        int rc = ensure_kv(d, fn, dcap);
        if (rc == RMU_OK) rc = grow(d->gen_ws, layout(nullptr));
        if (rc == RMU_OK) rc = grow(d->d_ids, T * sizeof(int32_t), token_rows(T) * sizeof(int32_t));
        if (rc == RMU_OK) rc = ensure_tokens(d, std::max(T, kRun), 1);
        if (rc != RMU_OK) return rc;
        layout(d->gen_ws.p);
        RMU_CUDA(cudaStreamWaitEvent(st, d->ws_done, 0));
        RMU_CUDA(cudaMemsetAsync(ints + kRun, 0, kRun * sizeof(int), st));
        return RMU_OK;
    }

    int operator()(const std::vector<int32_t>& seq, int k, int32_t* out) {
        const int S = static_cast<int>(seq.size()), p = S - 1, n = S - T, V = d->cfg.vocab_size;
        if (last_p >= 0) {
            // chain row last_p + j fed draft j: right while seq kept the drafts before it
            const int m = static_cast<int>(last.size());
            int kept = 0;
            while (kept < m && last_p + 1 + kept < S && seq[last_p + 1 + kept] == last[kept]) ++kept;
            dvalid = last_p + 1 + std::min(kept, std::max(m - 1, 0));
            if (schedule == RMU_ASSIST_HEURISTIC && m > 0) kcur = kept == m ? std::min(kcur + 2, kMaxDrafts) : std::max(kcur - 1, 1);
        }
        last_p = -1;
        last.clear();
        // no draft position reaches the draft's max_pos: the chain feeds positions p .. p + k - 1
        k = std::min({k, kcur, d->cfg.max_pos - p});
        if (k <= 0) return 0;
        const int cu_h[2] = {0, T};
        int rc = RMU_OK;
        if (!prefilled) {
            RMU_CUDA(cudaMemcpyAsync(d->d_ids.p, ids_h, T * sizeof(int32_t), cudaMemcpyHostToDevice, st));
            RMU_CUDA(cudaMemcpyAsync(d->span_cu, cu_h, sizeof(cu_h), cudaMemcpyHostToDevice, st));
            rc = run_qwen3(d, d->d_ids.as<int32_t>(), d->span_cu, 1, T, T, st, false, true);
            if (rc != RMU_OK) return rc;
            prefilled = true;
            dvalid = T;
        }
        for (; folded < seq.size(); ++folded) bits[seq[folded] >> 5] |= 1u << (seq[folded] & 31);
        RMU_CUDA(cudaMemcpyAsync(presence, bits.data(), words * sizeof(unsigned), cudaMemcpyHostToDevice, st));
        // catch-up: rows min(dvalid, p) .. p (the pending row always runs: its logits give draft 1)
        int hids[kRun], hpos[kRun], M = 0;
        for (int r0 = std::min(dvalid, p); r0 <= p && rc == RMU_OK; r0 += M) {
            M = std::min(kRun, p + 1 - r0);
            for (int j = 0; j < M; ++j) { hids[j] = seq[r0 + j]; hpos[j] = r0 + j; }
            RMU_CUDA(cudaMemcpyAsync(ints, hids, M * sizeof(int), cudaMemcpyHostToDevice, st));
            RMU_CUDA(cudaMemcpyAsync(d->POSI, hpos, M * sizeof(int), cudaMemcpyHostToDevice, st));
            rc = run_decode_rows(d, handle_kv(d), ints, M, ints + kRun, 0, r0 + M, part, st);
        }
        const float* row = d->PRE + static_cast<size_t>(M - 1) * d->cfg.hidden;
        for (int j = 1; j <= k && rc == RMU_OK; ++j) {
            if (j > 1) rc = run_decode_step(d, tok + j - 2, p + j - 1, part, st);
            if (rc == RMU_OK) rc = run_lm_head(d, row, 1, logits, st);
            if (rc == RMU_OK)
                rc = launch_sample(logits, V, presence, sa, -1.f, seed, static_cast<unsigned long long>(n + j - 1), tok + j - 1, st);
            row = d->PRE;
        }
        if (rc != RMU_OK) return rc;
        int flag = 0;
        RMU_CUDA(cudaMemcpyAsync(out, tok, k * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        RMU_CUDA(cudaMemcpyAsync(&flag, d->range_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
        RMU_CUDA(cudaStreamSynchronize(st));
        last_p = p;                                        // the catch-up rows stand: dvalid >= p + 1 next call
        if (flag) {
            RMU_CUDA(cudaMemsetAsync(d->range_flag, 0, sizeof(int), st));
            return 0;
        }
        // sample_kernel writes an id of [0, V) even from NaN logits; the target never reads one outside it regardless
        int m = 0;
        while (m < k && out[m] >= 0 && out[m] < V) ++m;
        last.assign(out, out + m);
        return m;
    }
};

int rmu_decoder_generate_assisted(rmu_encoder* e, rmu_encoder* draft, const int32_t* ids_h, int T, const rmu_sampling* s,
                                  uint64_t seed, int max_new_tokens, int num_tokens, int schedule, int32_t* out_h,
                                  int32_t* n_out, float* logits_h, int32_t* n_passes, int32_t* n_drafted, int32_t* n_kept,
                                  void* stream) {
    const std::string fn("rmu_decoder_generate_assisted");
    if (!e || !draft || !ids_h || !s || !out_h || !n_out || T < 1 || max_new_tokens < 1 || num_tokens < 0) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    if (schedule != RMU_ASSIST_CONSTANT && schedule != RMU_ASSIST_HEURISTIC) {
        set_error(fn + ": unknown schedule " + std::to_string(schedule) + " (RMU_ASSIST_CONSTANT or RMU_ASSIST_HEURISTIC)");
        return RMU_ERR_ARG;
    }
    if (draft == e) { set_error(fn + ": the draft must be another handle than the target"); return RMU_ERR_ARG; }
    int rc = check_generate(e, fn, ids_h, T, s);
    if (rc == RMU_OK) rc = check_generator(draft, fn + " (draft)");
    if (rc != RMU_OK) return rc;
    if (draft->cfg.vocab_size != e->cfg.vocab_size) {
        set_error(fn + ": the draft's vocab_size " + std::to_string(draft->cfg.vocab_size) + " differs from the target's " +
                  std::to_string(e->cfg.vocab_size) + ": the two models must share a tokenizer");
        return RMU_ERR_ARG;
    }
    if (draft->device != e->device) {
        set_error(fn + ": the draft is on device " + std::to_string(draft->device) + ", the target on device " +
                  std::to_string(e->device));
        return RMU_ERR_ARG;
    }
    std::scoped_lock lk(e->host_mu, e->mu, draft->host_mu, draft->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int k0 = std::min(num_tokens, kMaxDrafts);
    ModelDrafter md{draft, st, ids_h, T, std::min(T + max_new_tokens, draft->cfg.max_pos), schedule, k0, sample_args(*s), seed};
    if (k0 > 0) rc = md.setup(fn);
    if (rc != RMU_OK) return rc;
    const Drafter dr = [&](const std::vector<int32_t>& seq, int k, int32_t* out) { return md(seq, k, out); };
    // the heuristic schedule may grow k to 15: the loop's workspace is laid out for it
    const int kmax = k0 > 0 && schedule == RMU_ASSIST_HEURISTIC ? kMaxDrafts : k0;
    rc = generate_loop(e, fn, ids_h, T, s, seed, max_new_tokens, kmax, dr, out_h, n_out, logits_h, n_passes, stream,
                       n_drafted, n_kept);
    if (k0 > 0) {
        const cudaError_t err = cudaEventRecord(draft->ws_done, st);
        if (rc == RMU_OK && err != cudaSuccess) { set_error(fn + ": " + cudaGetErrorString(err)); rc = RMU_ERR_CUDA; }
    }
    return rc;
}

// The batch layout.  P = the prompts' longest common prefix, capped so that every prompt keeps one own token (0 when
// B = 1).  Per layer the KV cache holds the prefix at rows 0 .. P - 1 and prompt b's own keys (positions P ..) in rows
// P + b R + (k - P), R = the most own positions any prompt can reach.  The prefix runs once; the suffixes run as one
// varlen prefill at positions P + t (a one-token prompt of an NF4 handle runs alone, on the GEMV its own prefill takes);
// each decode step runs the live rows at M = live, decode attention over [prefix | own region].  Row b's tokens and
// logits are those of rmu_decoder_generate on prompt b with seeds_h[b] (DESIGN.md, "Batched decoding").
int rmu_decoder_generate_batch(rmu_encoder* e, const int32_t* ids_h, const int32_t* cu_h, int B, const rmu_sampling* s,
                               const uint64_t* seeds_h, int max_new_tokens, int32_t* out_h, int32_t* n_out_h,
                               float* logits_h, void* stream) {
    const std::string fn("rmu_decoder_generate_batch");
    if (!e || !ids_h || !cu_h || !s || !seeds_h || !out_h || !n_out_h || B < 1 || max_new_tokens < 1) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    // 0 until the call succeeds: any failure, refusal or CUDA error, leaves every count 0
    for (int b = 0; b < std::min(B, RMU_MAX_GENERATE_BATCH); ++b) n_out_h[b] = 0;
    if (B > RMU_MAX_GENERATE_BATCH) {
        set_error(fn + ": at most " + std::to_string(RMU_MAX_GENERATE_BATCH) + " prompts per call, got " + std::to_string(B));
        return RMU_ERR_ARG;
    }
    int rc = check_generator(e, fn);
    if (rc == RMU_OK) rc = check_prompts(e, fn, ids_h, cu_h, B);
    if (rc == RMU_OK) rc = check_sampling(fn, s);
    if (rc != RMU_OK) return rc;
    const rmu_bert_config& c = e->cfg;
    std::vector<int> Tb(B);
    for (int b = 0; b < B; ++b) Tb[b] = cu_h[b + 1] - cu_h[b];
    const int32_t* prompt0 = ids_h + cu_h[0];
    int P = B > 1 ? Tb[0] - 1 : 0;
    for (int b = 1; b < B; ++b) {
        P = std::min(P, Tb[b] - 1);
        const int32_t* pb = ids_h + cu_h[b];
        for (int i = 0; i < P; ++i)
            if (pb[i] != prompt0[i]) { P = i; break; }
    }
    // own positions: prompt b reaches at most min(T_b + max_new, max_pos) - 1
    int R = 1, most = 1;
    for (int b = 0; b < B; ++b) {
        const int end = std::min(Tb[b] + max_new_tokens, c.max_pos);
        R = std::max(R, end - P);
        most = std::max(most, end);
    }
    std::lock_guard<std::mutex> hg(e->host_mu);
    std::lock_guard<std::mutex> g(e->mu);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int V = c.vocab_size, nh = c.heads;
    // prefill runs: the prefix (prompt 0's first P tokens), then prefill_groups from token P of each prompt
    const int cu_prefix[2] = {cu_h[0], cu_h[0] + P};
    const std::vector<std::vector<int>> groups = prefill_groups(e, Tb);
    int suffix_rows = 0;                                 // the last group's run is the longest: a solo run has one row
    for (int b : groups.back()) suffix_rows += Tb[b] - P;
    const int rows_most = std::max({P, suffix_rows, B});
    // gen_ws: logits [B, V] | last hidden rows [B, H] | decode partials | presence [B, words] | seeds [B] | tokens [B] |
    // ints (ids, cu, shift of a prefill run; ids, shift, seq of a step)
    const size_t words = (static_cast<size_t>(V) + 31) / 32;
    float *logits, *last, *part;
    unsigned* presence;
    unsigned long long* seeds;
    int *tok, *ints;
    auto layout = [&](void* base) {
        Carve w(base);
        logits = w.take<float>(static_cast<size_t>(B) * V);
        last = w.take<float>(static_cast<size_t>(B) * c.hidden);
        part = w.take<float>(B * decode_part_floats(nh, most));
        presence = w.take<unsigned>(B * words);
        seeds = w.take<unsigned long long>(B);
        tok = w.take<int>(B);
        ints = w.take<int>(2 * static_cast<size_t>(rows_most) + B + 1 + 3 * static_cast<size_t>(B));
        return w.size;
    };
    rc = ensure_kv(e, fn, P + B * R);
    if (rc == RMU_OK) rc = grow(e->gen_ws, layout(nullptr));
    if (rc == RMU_OK) rc = ensure_tokens(e, rows_most, B);
    if (rc != RMU_OK) return rc;
    layout(e->gen_ws.p);
    std::vector<unsigned> bits(static_cast<size_t>(B) * words);
    for (int b = 0; b < B; ++b) prompt_bits(ids_h + cu_h[b], Tb[b], words, bits.data() + b * words);
    RMU_CUDA(cudaStreamWaitEvent(st, e->ws_done, 0));    // the activation workspace and gen_ws are shared by all callers
    RMU_CUDA(cudaMemsetAsync(e->range_flag, 0, sizeof(int), st));
    // pageable sources: each copy has taken its bytes when it returns
    RMU_CUDA(cudaMemcpyAsync(presence, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(seeds, seeds_h, static_cast<size_t>(B) * 8, cudaMemcpyHostToDevice, st));
    // one prefill run: ids | cu | shift into ints, positions into POSI
    auto prefill = [&](const PrefillRows& pr, int P0, bool gemv) -> int {
        const int n = pr.cu.back(), nb = static_cast<int>(pr.cu.size()) - 1;
        std::vector<int> packed(pr.ids);
        packed.insert(packed.end(), pr.cu.begin(), pr.cu.end());
        packed.insert(packed.end(), pr.shift.begin(), pr.shift.end());
        RMU_CUDA(cudaMemcpyAsync(ints, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, st));
        RMU_CUDA(cudaMemcpyAsync(e->POSI, pr.pos.data(), pr.pos.size() * 4, cudaMemcpyHostToDevice, st));
        return run_batch_prefill(e, handle_kv(e), ints, ints + n, ints + n + nb + 1, nb, n, pr.max_own, P0, gemv, st);
    };
    if (P > 0) rc = prefill(prefill_rows(ids_h, cu_prefix, {0}, 0, {0}), 0, false);
    for (const auto& g : groups) {
        std::vector<int> shift;
        for (int b : g) shift.push_back(b * R);
        const PrefillRows pr = prefill_rows(ids_h, cu_h, g, P, shift);
        if (rc == RMU_OK) rc = prefill(pr, P, e->nf4 && g.size() == 1 && Tb[g[0]] == 1);
        if (rc == RMU_OK) rc = gather_last(e, pr.cu, g.data(), last, st);
    }

    const SampleArgs sa = sample_args(*s);
    std::vector<int> live(B), n_b(B, 0), last_tok(B, 0);
    for (int b = 0; b < B; ++b) live[b] = b;
    const float* x_last = last;
    for (int step = 0; rc == RMU_OK && !live.empty(); ++step) {
        const int M = static_cast<int>(live.size());
        // ints: ids [M] | shift [M] | seq [M]; POSI: the positions of the tokens this step feeds
        std::vector<int> packed(3 * static_cast<size_t>(M)), hpos(M);
        for (int r = 0; r < M; ++r) {
            const int b = live[r];
            packed[r] = last_tok[b];
            packed[M + r] = b * R;
            packed[2 * M + r] = b;
            hpos[r] = Tb[b] + n_b[b] - 1;
        }
        RMU_CUDA(cudaMemcpyAsync(ints, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, st));
        if (step > 0) {
            int maxn = 0;
            for (int r = 0; r < M; ++r) maxn = std::max(maxn, hpos[r] + 1);
            RMU_CUDA(cudaMemcpyAsync(e->POSI, hpos.data(), hpos.size() * 4, cudaMemcpyHostToDevice, st));
            rc = run_decode_rows(e, handle_kv(e), ints, M, ints + M, P, maxn, part, st);
            x_last = e->PRE;
        }
        // logits for the M live rows (step 0: last[b] in prompt order), then the sampler
        if (rc == RMU_OK) rc = run_lm_head(e, x_last, M, logits, st);
        for (int r = 0; r < M && rc == RMU_OK && logits_h; ++r)
            RMU_CUDA(cudaMemcpyAsync(logits_h + (static_cast<size_t>(live[r]) * max_new_tokens + step) * V,
                                     logits + static_cast<size_t>(r) * V, static_cast<size_t>(V) * sizeof(float),
                                     cudaMemcpyDeviceToHost, st));
        SampleRows sr;
        sr.seq = ints + 2 * M;
        sr.seeds = seeds;
        sr.words = words;
        if (rc == RMU_OK) rc = launch_sample(logits, V, presence, sa, -1.f, 0ull, static_cast<unsigned long long>(step), tok, st, M, sr);
        if (rc != RMU_OK) break;
        std::vector<int> t_h(M);
        RMU_CUDA(cudaMemcpyAsync(t_h.data(), tok, static_cast<size_t>(M) * sizeof(int), cudaMemcpyDeviceToHost, st));
        rc = qwen3_check_range(e, st);        // synchronises st
        if (rc != RMU_OK) break;
        std::vector<int> next;
        for (int r = 0; r < M; ++r) {
            const int b = live[r];
            out_h[static_cast<size_t>(b) * max_new_tokens + n_b[b]++] = t_h[r];
            last_tok[b] = t_h[r];
            if (stop_status(*s, t_h[r], n_b[b], max_new_tokens, Tb[b], c.max_pos) == RMU_GEN_LIVE) next.push_back(b);
        }
        live.swap(next);
    }
    for (int b = 0; b < B; ++b) n_out_h[b] = rc == RMU_OK ? n_b[b] : 0;
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Continuous batching (DESIGN.md, "Continuous batching"): a decode session outlives one call.  Requests join it
// (rmu_decoder_session_add) and leave it (a stop, rmu_decoder_session_cancel) between steps; each step
// (rmu_decoder_session_step) runs every live row at M = live.  The session owns its KV cache, in the handle cache's
// layout; a request of T prompt tokens holds the region [base, base + min(T + max_new, max_pos)) and reads key k at
// row k + base (shift = base, P = 0).  Every entry point holds the handle's mu for its own duration only.
// ---------------------------------------------------------------------------------------------------

// The regions of a session's KV cache: the used ones by base; a gap is whatever lies between them, so a freed region
// merges with its free neighbours by construction.  Placement is first fit; past the last used region the cache grows,
// which moves no region, so every live row's shift stays valid.
struct KvRegions {
    std::map<int, int> used;                      // base -> rows
    int cap = 0;
    // the first gap of n rows; -1 when none fits, *need then the cap that fits n rows after the last used region
    int fit(int n, int* need) const {
        int at = 0;
        for (const auto& r : used) {
            if (r.first - at >= n) return at;
            at = r.first + r.second;
        }
        if (cap - at >= n) return at;
        *need = at + n;
        return -1;
    }
    // place n rows, growing cap when no gap fits -> the base
    int place(int n) {
        int need = 0;
        int base = fit(n, &need);
        if (base < 0) { cap = need; base = need - n; }
        used[base] = n;
        return base;
    }
};

struct rmu_gen_session {
    rmu_encoder* e = nullptr;
    KvRegions reg;
    void* kv = nullptr;                           // [L][4][kv_heads][reg.cap][128] halves
    // persistent device state, one entry per row slot: presence bits [16, words] (at state) | seeds [16] | settings
    // [16] | Philox steps [16]
    void* state = nullptr;
    size_t words = 0;
    unsigned long long *seeds = nullptr, *steps = nullptr;
    SampleArgs* args = nullptr;
    DevBuf ws;                                    // one call's scratch: logits, last rows, partials, tokens, ints
    struct Row {
        bool live = false;
        int base = 0, T = 0, n = 0, max_new = 0, last = 0;
        rmu_sampling s{};
    };
    Row rows[RMU_MAX_GENERATE_BATCH];
    cudaEvent_t done = nullptr;                   // the session's last use of its buffers
};

namespace {

KvView session_kv(rmu_gen_session* S) { return KvView{static_cast<__half*>(S->kv), S->reg.cap}; }
unsigned* session_presence(rmu_gen_session* S, int slot) {
    return static_cast<unsigned*>(S->state) + static_cast<size_t>(slot) * S->words;
}

// grow the session's cache to cap rows, each (layer, plane, head) block copied to the new pitch by one 2D copy
int session_grow(rmu_gen_session* S, int cap, cudaStream_t st) {
    rmu_encoder* e = S->e;
    const size_t blocks = static_cast<size_t>(e->cfg.layers) * 4 * e->qext.kv_heads, row = kQwenHD * sizeof(__half);
    void* p = nullptr;
    const cudaError_t err = cudaMalloc(&p, blocks * cap * row);
    if (err != cudaSuccess) {
        cudaGetLastError();
        set_error("cannot allocate " + std::to_string(blocks * cap * row) + " bytes of device memory: " +
                  cudaGetErrorString(err));
        return RMU_ERR_CUDA;
    }
    if (S->reg.cap > 0) {
        cudaError_t ce = cudaMemcpy2DAsync(p, cap * row, S->kv, S->reg.cap * row, S->reg.cap * row, blocks,
                                           cudaMemcpyDeviceToDevice, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
        if (ce != cudaSuccess) {                  // the old cache stays in place
            cudaFree(p);
            set_error(std::string("the session's KV cache copy failed: ") + cudaGetErrorString(ce));
            return RMU_ERR_CUDA;
        }
    }
    cudaFree(S->kv);
    S->kv = p;
    S->reg.cap = cap;
    return RMU_OK;
}

// the sampler over M rows whose slots are seq (device [M]), each with its slot's bits, seed, settings and step
int session_sample(rmu_gen_session* S, float* logits, int M, const int* seq, int* tok, cudaStream_t st) {
    SampleRows sr;
    sr.seq = seq;
    sr.seeds = S->seeds;
    sr.words = S->words;
    sr.args = S->args;
    sr.steps = S->steps;
    return launch_sample(logits, S->e->cfg.vocab_size, static_cast<unsigned*>(S->state), SampleArgs{}, -1.f, 0ull, 0ull,
                         tok, st, M, sr);
}

// One pass over the slots `slots` (row r = slots[r]): with T null a decode step, each row feeding its last token at
// position T + n - 1; else the prefill of new requests, prompt r = ids_h[cu_h[req[r]] ..) (one varlen run; gemv: one
// one-token prompt on the decode GEMV).  Then the LM head, logits to logits_h (nullable, [M, V]), the sampler, the tokens
// to t_h.  *raised <- the range flag; when raised, the presence bits are restored to what they were before the pass.
int session_pass(rmu_gen_session* S, const std::vector<int>& slots, const int32_t* ids_h, const int32_t* cu_h,
                 const std::vector<int>* req, bool gemv, float* logits_h, int* t_h, bool* raised, cudaStream_t st) {
    rmu_encoder* e = S->e;
    const rmu_bert_config& c = e->cfg;
    const int M = static_cast<int>(slots.size()), V = c.vocab_size;
    std::vector<int> base;
    for (int q : slots) base.push_back(S->rows[q].base);
    PrefillRows pr;                               // a decode step's rows in the same fields, with cu [0]
    int maxn = 0;
    if (req) pr = prefill_rows(ids_h, cu_h, *req, 0, base);
    for (int r = 0; r < M && !req; ++r) {
        const rmu_gen_session::Row& w = S->rows[slots[r]];
        pr.ids.push_back(w.last);
        pr.pos.push_back(w.T + w.n - 1);
        pr.shift.push_back(base[r]);
        maxn = std::max(maxn, w.T + w.n);
    }
    const int rows = static_cast<int>(pr.ids.size());
    std::vector<int> packed(pr.ids);
    packed.insert(packed.end(), pr.shift.begin(), pr.shift.end());
    packed.insert(packed.end(), slots.begin(), slots.end());
    packed.insert(packed.end(), pr.cu.begin(), pr.cu.end());
    // S->ws: logits [16, V] | last hidden rows [16, H] | decode partials | presence backup [16, words] | tokens [16] |
    // ints (packed).  The partials are sized for 16 rows over the longest region in the session, and the buffer grows
    // with half again as much headroom, so a reply's steps do not re-grow it as its keys pass each split.
    const size_t R = std::max(M, RMU_MAX_GENERATE_BATCH);
    int longest = 1;
    for (const auto& u : S->reg.used) longest = std::max(longest, u.second);
    const size_t part_f = std::max(req ? 0 : M * decode_part_floats(c.heads, maxn),
                                   RMU_MAX_GENERATE_BATCH * decode_part_floats(c.heads, longest));
    float *logits, *last, *part;
    unsigned* backup;
    int *tok, *ints;
    auto layout = [&](void* p) {
        Carve b(p);
        logits = b.take<float>(R * V);
        last = b.take<float>(R * c.hidden);
        part = b.take<float>(part_f);
        backup = b.take<unsigned>(RMU_MAX_GENERATE_BATCH * S->words);
        tok = b.take<int>(RMU_MAX_GENERATE_BATCH);
        ints = b.take<int>(packed.size());
        return b.size;
    };
    const size_t need = layout(nullptr);
    int rc = grow(S->ws, need, need + need / 2);
    if (rc == RMU_OK) rc = ensure_tokens(e, rows, M);
    if (rc != RMU_OK) return rc;
    layout(S->ws.p);
    int* shift = ints + rows;
    int* seq_off = shift + rows;
    int* cu = seq_off + M;
    RMU_CUDA(cudaMemsetAsync(e->range_flag, 0, sizeof(int), st));
    // pageable sources: each copy has taken its bytes when it returns
    RMU_CUDA(cudaMemcpyAsync(ints, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(e->POSI, pr.pos.data(), pr.pos.size() * 4, cudaMemcpyHostToDevice, st));
    unsigned long long steps[RMU_MAX_GENERATE_BATCH];             // every slot's Philox step: its tokens so far
    for (int i = 0; i < RMU_MAX_GENERATE_BATCH; ++i) steps[i] = static_cast<unsigned long long>(S->rows[i].n);
    RMU_CUDA(cudaMemcpyAsync(S->steps, steps, sizeof(steps), cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(backup, S->state, RMU_MAX_GENERATE_BATCH * S->words * 4, cudaMemcpyDeviceToDevice, st));
    const KvView kvv = session_kv(S);
    const float* x = e->PRE;
    if (req) {
        rc = run_batch_prefill(e, kvv, ints, cu, shift, M, rows, pr.max_own, 0, gemv, st);
        if (rc == RMU_OK) rc = gather_last(e, pr.cu, nullptr, last, st);
        x = last;
    } else {
        rc = run_decode_rows(e, kvv, ints, M, shift, 0, maxn, part, st);
    }
    if (rc == RMU_OK) rc = run_lm_head(e, x, M, logits, st);
    if (rc == RMU_OK && logits_h)
        RMU_CUDA(cudaMemcpyAsync(logits_h, logits, static_cast<size_t>(M) * V * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (rc == RMU_OK) rc = session_sample(S, logits, M, seq_off, tok, st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(t_h, tok, static_cast<size_t>(M) * sizeof(int), cudaMemcpyDeviceToHost, st));
    rc = read_range(e, raised, st);               // synchronises st
    if (rc == RMU_OK && *raised)
        RMU_CUDA(cudaMemcpyAsync(S->state, backup, RMU_MAX_GENERATE_BATCH * S->words * 4, cudaMemcpyDeviceToDevice, st));
    return rc;
}

void release_row(rmu_gen_session* S, int slot) {
    S->reg.used.erase(S->rows[slot].base);
    S->rows[slot].live = false;
}

// the row in slot q after a pass gave it token t, or err when its own redo raised the range flag: its status, the row
// released when it stops
int finish_row(rmu_gen_session* S, int q, int t, int err) {
    rmu_gen_session::Row& w = S->rows[q];
    w.last = t;
    const int status = err != RMU_OK ? err : stop_status(w.s, t, ++w.n, w.max_new, w.T, S->e->cfg.max_pos);
    if (status != RMU_GEN_LIVE) release_row(S, q);
    return status;
}

// waits on the handle's workspace and the session's last use on st
int session_begin(rmu_gen_session* S, cudaStream_t st) {
    RMU_CUDA(cudaStreamWaitEvent(st, S->e->ws_done, 0));
    RMU_CUDA(cudaStreamWaitEvent(st, S->done, 0));
    return RMU_OK;
}

int session_end(rmu_gen_session* S, cudaStream_t st) {
    RMU_CUDA(cudaEventRecord(S->done, st));
    RMU_CUDA(cudaEventRecord(S->e->ws_done, st));
    return RMU_OK;
}

}  // namespace

extern "C" {

int rmu_decoder_session_create(rmu_encoder* e, rmu_gen_session** out) {
    const std::string fn("rmu_decoder_session_create");
    if (!e || !out) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    *out = nullptr;
    int rc = check_decoder(e, fn);
    if (rc == RMU_OK) rc = check_nf4_intact(e, fn);
    if (rc != RMU_OK) return rc;
    std::lock_guard<std::mutex> g(e->mu);
    rmu_gen_session* S = new rmu_gen_session();
    S->e = e;
    S->words = (static_cast<size_t>(e->cfg.vocab_size) + 31) / 32;
    auto layout = [S](void* base) {
        Carve b(base);
        b.take<unsigned>(RMU_MAX_GENERATE_BATCH * S->words);
        S->seeds = b.take<unsigned long long>(RMU_MAX_GENERATE_BATCH);
        S->args = b.take<SampleArgs>(RMU_MAX_GENERATE_BATCH);
        S->steps = b.take<unsigned long long>(RMU_MAX_GENERATE_BATCH);
        return b.size;
    };
    const size_t bytes = layout(nullptr);
    cudaError_t err = cudaSetDevice(e->device);
    if (err == cudaSuccess) err = cudaMalloc(&S->state, bytes);
    if (err == cudaSuccess) layout(S->state);
    if (err == cudaSuccess) err = cudaEventCreateWithFlags(&S->done, cudaEventDisableTiming);
    if (err == cudaSuccess) err = cudaMemset(S->state, 0, bytes);
    if (err != cudaSuccess) {
        cudaGetLastError();
        set_error(fn + ": " + cudaGetErrorString(err));
        cudaFree(S->state);
        if (S->done) cudaEventDestroy(S->done);
        delete S;
        return RMU_ERR_CUDA;
    }
    *out = S;
    return RMU_OK;
}

void rmu_decoder_session_destroy(rmu_gen_session* S) {
    if (!S) return;
    {
        std::lock_guard<std::mutex> g(S->e->mu);
        cudaEventSynchronize(S->done);
        cudaFree(S->kv);
        cudaFree(S->state);
        S->ws.release();
        cudaEventDestroy(S->done);
    }
    delete S;
}

int rmu_decoder_session_add(rmu_gen_session* S, const int32_t* ids_h, const int32_t* cu_h, int B, const rmu_sampling* s_h,
                            const uint64_t* seeds_h, const int32_t* max_new_h, int32_t* slot_h, int32_t* tok_h,
                            int32_t* status_h, float* logits_h, void* stream) {
    const std::string fn("rmu_decoder_session_add");
    if (!S || !ids_h || !cu_h || !s_h || !seeds_h || !max_new_h || !slot_h || !tok_h || !status_h || B < 1 ||
        B > RMU_MAX_GENERATE_BATCH) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    rmu_encoder* e = S->e;
    int rc = check_generator(e, fn);
    if (rc == RMU_OK) rc = check_prompts(e, fn, ids_h, cu_h, B);
    if (rc != RMU_OK) return rc;
    const rmu_bert_config& c = e->cfg;
    std::vector<int> Tb(B), nrows(B);
    for (int b = 0; b < B; ++b) {
        if (max_new_h[b] < 1) { set_error(fn + ": max_new_tokens must be at least 1"); return RMU_ERR_ARG; }
        rc = check_sampling(fn, s_h + b);
        if (rc != RMU_OK) return rc;
        Tb[b] = cu_h[b + 1] - cu_h[b];
        nrows[b] = static_cast<int>(std::min<int64_t>(static_cast<int64_t>(Tb[b]) + max_new_h[b], c.max_pos));
    }
    std::lock_guard<std::mutex> g(e->mu);
    std::vector<int> free_slots;
    for (int i = 0; i < RMU_MAX_GENERATE_BATCH; ++i)
        if (!S->rows[i].live) free_slots.push_back(i);
    int live = RMU_MAX_GENERATE_BATCH - static_cast<int>(free_slots.size());
    if (static_cast<int>(free_slots.size()) < B) {
        set_error(fn + ": " + std::to_string(live) + " rows are live and " + std::to_string(B) + " more do not fit (at most " +
                  std::to_string(RMU_MAX_GENERATE_BATCH) + ")");
        return RMU_ERR_BUSY;
    }
    KvRegions reg = S->reg;
    std::vector<int> base(B);
    for (int b = 0; b < B; ++b) base[b] = reg.place(nrows[b]);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RMU_CUDA(cudaSetDevice(e->device));
    rc = session_begin(S, st);
    if (rc != RMU_OK) return rc;
    if (reg.cap > S->reg.cap) {
        rc = session_grow(S, reg.cap, st);
        if (rc != RMU_OK) {
            if (live > 0) {
                set_error(fn + ": the session's KV cache cannot grow to " + std::to_string(reg.cap) + " positions while " +
                          std::to_string(live) + " rows are live: " + rmu_last_error());
                return RMU_ERR_BUSY;
            }
            set_error(fn + ": the KV cache for " + std::to_string(reg.cap) + " positions: " + rmu_last_error());
            return rc;
        }
    }
    S->reg = reg;
    std::vector<int> slots(B);
    std::vector<unsigned> bits(S->words);
    for (int b = 0; b < B; ++b) {
        const int q = slots[b] = free_slots[b];
        rmu_gen_session::Row& w = S->rows[q];
        w = rmu_gen_session::Row{};
        w.live = true;
        w.base = base[b];
        w.T = Tb[b];
        w.max_new = max_new_h[b];
        w.s = s_h[b];
    }
    // from here on a failure releases the new rows (a grown cache stays grown)
    auto settings = [&]() -> int {
        for (int b = 0; b < B; ++b) {
            const SampleArgs sa = sample_args(s_h[b]);
            RMU_CUDA(cudaMemcpyAsync(S->seeds + slots[b], seeds_h + b, 8, cudaMemcpyHostToDevice, st));
            RMU_CUDA(cudaMemcpyAsync(S->args + slots[b], &sa, sizeof(SampleArgs), cudaMemcpyHostToDevice, st));
        }
        return RMU_OK;
    };
    rc = settings();
    // the prompt's presence bits of request b's slot
    auto upload_bits = [&](int b) -> int {
        prompt_bits(ids_h + cu_h[b], Tb[b], S->words, bits.data());
        RMU_CUDA(cudaMemcpyAsync(session_presence(S, slots[b]), bits.data(), S->words * 4, cudaMemcpyHostToDevice, st));
        return RMU_OK;
    };
    for (int b = 0; b < B && rc == RMU_OK; ++b) rc = upload_bits(b);
    // prefill groups as rmu_decoder_generate_batch runs them
    const int V = c.vocab_size;
    std::vector<int> t_h(B, 0), err(B, RMU_OK);
    const std::vector<std::vector<int>> groups = prefill_groups(e, Tb);
    auto run = [&](const std::vector<int>& g, bool* raised) -> int {
        std::vector<int> sl, tt(g.size());
        for (int b : g) sl.push_back(slots[b]);
        const bool gemv = e->nf4 && g.size() == 1 && Tb[g[0]] == 1;
        std::vector<float> lg(logits_h ? g.size() * static_cast<size_t>(V) : 0);
        int r = session_pass(S, sl, ids_h, cu_h, &g, gemv, logits_h ? lg.data() : nullptr, tt.data(), raised, st);
        if (r != RMU_OK || *raised) return r;
        for (size_t i = 0; i < g.size(); ++i) {
            t_h[g[i]] = tt[i];
            if (logits_h) std::copy(lg.begin() + i * V, lg.begin() + (i + 1) * V, logits_h + static_cast<size_t>(g[i]) * V);
        }
        return RMU_OK;
    };
    for (const auto& gr : groups) {
        if (rc != RMU_OK) break;
        bool raised = false;
        rc = run(gr, &raised);
        if (rc != RMU_OK || !raised) continue;
        // one request's activations left fp16's range: redo them one at a time, and end only those whose own run raises
        // the flag too
        for (int b : gr) {
            if (gr.size() > 1) {
                rc = upload_bits(b);
                if (rc == RMU_OK) rc = run({b}, &raised);
                if (rc != RMU_OK) break;
            }
            if (raised) err[b] = RMU_ERR_RANGE;
        }
    }
    if (rc != RMU_OK) {
        for (int b = 0; b < B; ++b) release_row(S, slots[b]);
        return rc;
    }
    for (int b = 0; b < B; ++b) {
        tok_h[b] = t_h[b];
        status_h[b] = finish_row(S, slots[b], t_h[b], err[b]);
        slot_h[b] = status_h[b] == RMU_GEN_LIVE ? slots[b] : -1;
    }
    return session_end(S, st);
}

int rmu_decoder_session_step(rmu_gen_session* S, int32_t* slot_h, int32_t* tok_h, int32_t* status_h, int32_t* n_h,
                             float* logits_h, void* stream) {
    const std::string fn("rmu_decoder_session_step");
    if (!S || !slot_h || !tok_h || !status_h || !n_h) { set_error(fn + ": bad argument"); return RMU_ERR_ARG; }
    *n_h = 0;
    rmu_encoder* e = S->e;
    std::lock_guard<std::mutex> g(e->mu);
    std::vector<int> slots;
    for (int i = 0; i < RMU_MAX_GENERATE_BATCH; ++i)
        if (S->rows[i].live) slots.push_back(i);
    if (slots.empty()) return RMU_OK;
    const int M = static_cast<int>(slots.size()), V = e->cfg.vocab_size;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = RMU_OK;
    const cudaError_t de = cudaSetDevice(e->device);
    if (de != cudaSuccess) { set_error(fn + ": " + cudaGetErrorString(de)); rc = RMU_ERR_CUDA; }
    if (rc == RMU_OK) rc = session_begin(S, st);
    std::vector<int> t_h(M, 0), err(M, RMU_OK);
    bool raised = false;
    if (rc == RMU_OK) rc = session_pass(S, slots, nullptr, nullptr, nullptr, true, logits_h, t_h.data(), &raised, st);
    if (rc == RMU_OK && raised) {
        // redo the rows one at a time; only a row whose own step raises the flag ends, with RMU_ERR_RANGE
        for (int r = 0; r < M && rc == RMU_OK; ++r) {
            if (M > 1)
                rc = session_pass(S, {slots[r]}, nullptr, nullptr, nullptr, true,
                                  logits_h ? logits_h + static_cast<size_t>(r) * V : nullptr, &t_h[r], &raised, st);
            if (raised) err[r] = RMU_ERR_RANGE;
        }
    }
    if (rc != RMU_OK) {
        // a failed step leaves its rows without a consistent state: every one of them is released
        for (int q : slots) release_row(S, q);
        return rc;
    }
    for (int r = 0; r < M; ++r) {
        slot_h[r] = slots[r];
        tok_h[r] = t_h[r];
        status_h[r] = finish_row(S, slots[r], t_h[r], err[r]);
    }
    *n_h = M;
    return session_end(S, st);
}

int rmu_decoder_session_cancel(rmu_gen_session* S, int slot) {
    if (!S || slot < 0 || slot >= RMU_MAX_GENERATE_BATCH) {
        set_error("rmu_decoder_session_cancel: bad argument");
        return RMU_ERR_ARG;
    }
    std::lock_guard<std::mutex> g(S->e->mu);
    if (!S->rows[slot].live) { set_error("rmu_decoder_session_cancel: row " + std::to_string(slot) + " is not live"); return RMU_ERR_ARG; }
    release_row(S, slot);
    return RMU_OK;
}

int rmu_decoder_session_info(rmu_gen_session* S, int32_t* live, int32_t* cap_positions, uint32_t* live_mask) {
    if (!S || !live || !cap_positions) { set_error("rmu_decoder_session_info: bad argument"); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> g(S->e->mu);
    int n = 0;
    uint32_t mask = 0;
    for (int i = 0; i < RMU_MAX_GENERATE_BATCH; ++i) {
        n += S->rows[i].live ? 1 : 0;
        mask |= S->rows[i].live ? 1u << i : 0u;
    }
    *live = n;
    *cap_positions = S->reg.cap;
    if (live_mask) *live_mask = mask;
    return RMU_OK;
}

int rmu_debug_kv_regions(const int32_t* ops, int n, int32_t* out) {
    if (!ops || !out || n < 0) { set_error("rmu_debug_kv_regions: bad argument"); return RMU_ERR_ARG; }
    KvRegions reg;
    for (int i = 0; i < n; ++i) {
        if (ops[i] > 0) {
            out[2 * i] = reg.place(ops[i]);
        } else {
            out[2 * i] = reg.used.erase(-ops[i]) ? 0 : -1;
        }
        out[2 * i + 1] = reg.cap;
    }
    return RMU_OK;
}

}  // extern "C"

// ---- ColBERT: the encoder without a head, `linear` on the last hidden state, per-token normalisation, MaxSim
struct rmu_colbert {
    rmu_encoder* enc = nullptr;
    int dim = 0, dpad = 0;                // dpad: dim rounded up to E1's 128-column tile (zero rows of `linear`)
    SplitOperand lin;                     // linear [dpad, H] as split planes (allocations owned by enc)
    float* zero_bias = nullptr;           // [dpad]
    DevBuf proj;                          // [rows, dpad] fp32 projections: workspace, used under enc->mu
    // staging of rmu_colbert_score_host, owned by host_mu
    DevBuf s_qids, s_qcu, s_qnk, s_dids, s_dcu, s_dkeep, s_qv, s_dv, s_pq, s_pd, s_out;
    std::mutex host_mu;
};

// token vectors of a ragged batch -> out [T, dim]: the encoder (keys limited by nkeys when given), E1 mode 0 with
// `linear` and a zero bias on the last hidden state's split planes -> proj fp32, then C1
static int colbert_vectors(rmu_colbert* cb, const int32_t* ids, const int32_t* cu, const int32_t* nkeys, const uint8_t* keep,
                           int B, int T, int max_seqlen, float* out, cudaStream_t st) {
    rmu_encoder* e = cb->enc;
    std::lock_guard<std::mutex> g(e->mu);
    const size_t row = cb->dpad * sizeof(float);
    int rc = grow(cb->proj, T * row, token_rows(T) * row);
    if (rc == RMU_OK) rc = run_encoder(e, ids, nullptr, cu, B, T, max_seqlen, false, st, nkeys);
    if (rc != RMU_OK) return rc;
    GemmParams g2{};
    g2.M = T; g2.N = cb->dpad; g2.K = e->cfg.hidden; g2.bias = cb->zero_bias; g2.out_f32 = cb->proj.as<float>();
    rc = launch_gemm(GEMM_BIAS_F32, e->X, cb->lin, g2, e->sms, st);
    if (rc != RMU_OK) return rc;
    rc = launch_colbert_normalize(cb->proj.as<float>(), T, cb->dpad, cb->dim, keep, out, st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaEventRecord(e->ws_done, st));
    return RMU_OK;
}

extern "C" {

int rmu_colbert_create(const rmu_bert_config* cfg, const float* const* w, int n_weights, const float* linear_h, int dim,
                       rmu_colbert** out) {
    if (!cfg || !w || !linear_h || !out || dim <= 0 || cfg->hidden <= 0) {
        set_error("rmu_colbert_create: bad argument");
        return RMU_ERR_ARG;
    }
    if (dim > 128 && dim % 128 != 0) {
        set_error("rmu_colbert_create: dim must be at most 128 or a multiple of 128");
        return RMU_ERR_UNSUPPORTED;
    }
    if (cfg->rel_buckets != 0) {
        set_error("rmu_colbert_create: a relative attention bias is not supported with ColBERT's key limit");
        return RMU_ERR_UNSUPPORTED;
    }
    const int H = cfg->hidden;
    const size_t n = static_cast<size_t>(dim) * H;
    int rc = check_split_range("rmu_colbert_create", "linear", linear_h, n);
    if (rc != RMU_OK) return rc;
    rmu_encoder* enc = nullptr;
    rc = rmu_encoder_create(cfg, w, n_weights, 0, &enc);
    if (rc != RMU_OK) return rc;
    rmu_colbert* cb = new rmu_colbert();
    cb->enc = enc;
    cb->dim = dim;
    cb->dpad = (dim + 127) / 128 * 128;
    std::vector<float> pad(static_cast<size_t>(cb->dpad) * H, 0.f);
    std::copy(linear_h, linear_h + n, pad.begin());
    rc = upload_split(enc, &cb->lin, {pad.data()}, cb->dpad, H);
    std::vector<float> zeros(cb->dpad, 0.f);
    if (rc == RMU_OK) rc = upload(enc, &cb->zero_bias, zeros.data(), zeros.size());
    if (rc != RMU_OK) { rmu_colbert_destroy(cb); return rc; }
    *out = cb;
    return RMU_OK;
}

void rmu_colbert_destroy(rmu_colbert* cb) {
    if (!cb) return;
    cudaDeviceSynchronize();
    for (DevBuf* b : {&cb->proj, &cb->s_qids, &cb->s_qcu, &cb->s_qnk, &cb->s_dids, &cb->s_dcu, &cb->s_dkeep, &cb->s_qv,
                      &cb->s_dv, &cb->s_pq, &cb->s_pd, &cb->s_out})
        b->release();
    rmu_encoder_destroy(cb->enc);
    delete cb;
}

int rmu_colbert_dim(const rmu_colbert* cb) { return cb ? cb->dim : 0; }

int rmu_colbert_vectors(rmu_colbert* cb, const int32_t* ids, const int32_t* cu, const int32_t* nkeys, const uint8_t* keep,
                        int B, int T, int max_seqlen, float* out, void* stream) {
    int rc = check_batch(cb ? cb->enc : nullptr, ids, cu, B, T, out);
    if (rc != RMU_OK) return rc;
    return colbert_vectors(cb, ids, cu, nkeys, keep, B, T, max_seqlen, out, static_cast<cudaStream_t>(stream));
}

int rmu_colbert_maxsim(const float* q, const int32_t* q_cu, const float* d, const int32_t* d_cu, const uint8_t* d_keep,
                       int dim, const int32_t* pair_q, const int32_t* pair_d, int n_pairs, float* out, void* stream) {
    if (!q || !q_cu || !d || !d_cu || dim <= 0 || n_pairs < 0 || (n_pairs > 0 && (!pair_q || !pair_d || !out))) {
        set_error("rmu_colbert_maxsim: bad argument");
        return RMU_ERR_ARG;
    }
    return launch_colbert_maxsim(q, q_cu, d, d_cu, d_keep, dim, pair_q, pair_d, n_pairs, out, static_cast<cudaStream_t>(stream));
}

int rmu_colbert_score_host(rmu_colbert* cb, const int32_t* q_ids_h, const int32_t* q_cu_h, const int32_t* q_nkeys_h, int nq,
                           int q_tokens, const int32_t* d_ids_h, const int32_t* d_cu_h, const uint8_t* d_keep_h, int nd,
                           int d_tokens, const int32_t* pair_q_h, const int32_t* pair_d_h, int n_pairs,
                           int max_tokens_per_batch, float* out_h, void* stream) {
    if (!cb || !q_ids_h || !q_cu_h || !d_ids_h || !d_cu_h || !pair_q_h || !pair_d_h || !out_h || nq <= 0 || q_tokens <= 0 ||
        nd <= 0 || d_tokens <= 0 || n_pairs <= 0 || max_tokens_per_batch <= 0 || q_cu_h[0] != 0 || q_cu_h[nq] != q_tokens ||
        d_cu_h[0] != 0 || d_cu_h[nd] != d_tokens) {
        set_error("rmu_colbert_score_host: bad argument");
        return RMU_ERR_ARG;
    }
    for (int p = 0; p < n_pairs; ++p) {
        if (pair_q_h[p] < 0 || pair_q_h[p] >= nq || pair_d_h[p] < 0 || pair_d_h[p] >= nd) {
            set_error("rmu_colbert_score_host: pair index out of range");
            return RMU_ERR_ARG;
        }
    }
    int q_max = 0;
    for (int b = 0; b < nq; ++b) {
        if (q_cu_h[b + 1] < q_cu_h[b]) { set_error("rmu_colbert_score_host: q_cu must be non-decreasing"); return RMU_ERR_ARG; }
        q_max = std::max(q_max, q_cu_h[b + 1] - q_cu_h[b]);
    }
    for (int b = 0; b < nd; ++b) {
        const int t0 = d_cu_h[b], t1 = d_cu_h[b + 1];
        if (t1 < t0) { set_error("rmu_colbert_score_host: d_cu must be non-decreasing"); return RMU_ERR_ARG; }
        bool any = false;
        for (int t = t0; t < t1 && !any; ++t) any = d_keep_h == nullptr || d_keep_h[t] != 0;
        if (!any) { set_error("rmu_colbert_score_host: a document has no kept token"); return RMU_ERR_ARG; }
    }
    // document runs of at most max_tokens_per_batch tokens (a longer document runs alone), each with its own cu from 0
    std::vector<int> run_start{0}, run_cu;
    for (int s = 0; s < nd;) {
        int e = s + 1;
        while (e < nd && d_cu_h[e + 1] - d_cu_h[s] <= max_tokens_per_batch) ++e;
        for (int b = s; b <= e; ++b) run_cu.push_back(d_cu_h[b] - d_cu_h[s]);
        run_start.push_back(e);
        s = e;
    }
    const int dim = cb->dim;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::lock_guard<std::mutex> hg(cb->host_mu);
    int rc = RMU_OK;
    const size_t i4 = sizeof(int32_t);
    for (auto& [buf, bytes] : std::initializer_list<std::pair<DevBuf*, size_t>>{
             {&cb->s_qids, q_tokens * i4}, {&cb->s_qcu, (nq + 1) * i4}, {&cb->s_qnk, nq * i4}, {&cb->s_dids, d_tokens * i4},
             {&cb->s_dcu, (run_cu.size() + nd + 1) * i4}, {&cb->s_dkeep, static_cast<size_t>(d_tokens)},
             {&cb->s_qv, static_cast<size_t>(q_tokens) * dim * sizeof(float)},
             {&cb->s_dv, static_cast<size_t>(d_tokens) * dim * sizeof(float)}, {&cb->s_pq, n_pairs * i4},
             {&cb->s_pd, n_pairs * i4}, {&cb->s_out, n_pairs * sizeof(float)}}) {
        if (rc == RMU_OK) rc = grow(*buf, bytes, std::max<size_t>(bytes + bytes / 2, 4096));
    }
    if (rc != RMU_OK) return rc;
    auto* qids = static_cast<int32_t*>(cb->s_qids.p);
    auto* qcu = static_cast<int32_t*>(cb->s_qcu.p);
    auto* qnk = static_cast<int32_t*>(cb->s_qnk.p);
    auto* dids = static_cast<int32_t*>(cb->s_dids.p);
    auto* dcu = static_cast<int32_t*>(cb->s_dcu.p);         // [nd + 1] absolute, then the runs' own cu arrays
    auto* dkeep = static_cast<uint8_t*>(cb->s_dkeep.p);
    auto* qv = static_cast<float*>(cb->s_qv.p);
    auto* dv = static_cast<float*>(cb->s_dv.p);
    RMU_CUDA(cudaMemcpyAsync(qids, q_ids_h, q_tokens * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(qcu, q_cu_h, (nq + 1) * i4, cudaMemcpyHostToDevice, st));
    if (q_nkeys_h) RMU_CUDA(cudaMemcpyAsync(qnk, q_nkeys_h, nq * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(dids, d_ids_h, d_tokens * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(dcu, d_cu_h, (nd + 1) * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(dcu + nd + 1, run_cu.data(), run_cu.size() * i4, cudaMemcpyHostToDevice, st));
    if (d_keep_h) RMU_CUDA(cudaMemcpyAsync(dkeep, d_keep_h, d_tokens, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(cb->s_pq.p, pair_q_h, n_pairs * i4, cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(cb->s_pd.p, pair_d_h, n_pairs * i4, cudaMemcpyHostToDevice, st));
    rc = colbert_vectors(cb, qids, qcu, q_nkeys_h ? qnk : nullptr, nullptr, nq, q_tokens, q_max, qv, st);
    size_t cu_off = nd + 1;
    for (size_t r = 0; r + 1 < run_start.size() && rc == RMU_OK; ++r) {
        const int s = run_start[r], e = run_start[r + 1];
        const int t0 = d_cu_h[s], t1 = d_cu_h[e];
        int mx = 0;
        for (int b = s; b < e; ++b) mx = std::max(mx, d_cu_h[b + 1] - d_cu_h[b]);
        if (t1 > t0)
            rc = colbert_vectors(cb, dids + t0, dcu + cu_off, nullptr, d_keep_h ? dkeep + t0 : nullptr, e - s, t1 - t0, mx,
                                 dv + static_cast<size_t>(t0) * dim, st);
        cu_off += e - s + 1;
    }
    if (rc == RMU_OK)
        rc = launch_colbert_maxsim(qv, qcu, dv, dcu, d_keep_h ? dkeep : nullptr, dim, static_cast<int32_t*>(cb->s_pq.p),
                                   static_cast<int32_t*>(cb->s_pd.p), n_pairs, static_cast<float*>(cb->s_out.p), st);
    if (rc != RMU_OK) { cudaStreamSynchronize(st); return rc; }
    RMU_CUDA(cudaMemcpyAsync(out_h, cb->s_out.p, n_pairs * sizeof(float), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    return RMU_OK;
}

int rmu_debug_attention_keys(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, const int32_t* nkeys, int B,
                             int H, int heads, int max_seqlen, int warps, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !nkeys || !ctx_hi || !ctx_lo || B <= 0 || heads <= 0 || H <= 0 || max_seqlen <= 0) {
        set_error("rmu_debug_attention_keys: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % heads != 0 || (H / heads != 32 && H / heads != 64)) {
        set_error("rmu_debug_attention_keys: head_dim must be 32 or 64");
        return RMU_ERR_UNSUPPORTED;
    }
    if (warps != kAttWarps) { set_error("rmu_debug_attention_keys: warps must be 10"); return RMU_ERR_ARG; }
    return launch_attention(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), nullptr, nullptr,
                            cu, B, H, heads, max_seqlen, reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo),
                            static_cast<cudaStream_t>(stream), nullptr, nkeys);
}

// ---- kernel-level test entry points: the launchers run_encoder uses, on caller-owned planes
int rmu_debug_attention(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, int B, int H, int heads,
                        int max_seqlen, int warps, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !ctx_hi || !ctx_lo || B <= 0 || heads <= 0 || H <= 0 || max_seqlen <= 0) {
        set_error("rmu_debug_attention: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % heads != 0 || (H / heads != 32 && H / heads != 64)) {
        set_error("rmu_debug_attention: head_dim must be 32 or 64");
        return RMU_ERR_UNSUPPORTED;
    }
    if (warps != kAttWarps) { set_error("rmu_debug_attention: warps must be 10"); return RMU_ERR_ARG; }
    return launch_attention(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), nullptr, nullptr,
                            cu, B, H, heads, max_seqlen, reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo),
                            static_cast<cudaStream_t>(stream));
}

int rmu_debug_layernorm(const float* pre, int T, int H, const float* gamma, const float* beta, float eps,
                        uint16_t* out_hi, uint16_t* out_lo, void* stream) {
    if (!pre || !gamma || !beta || !out_hi || !out_lo || T <= 0 || H <= 0) {
        set_error("rmu_debug_layernorm: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % 128 != 0 || H > 32 * kMaxPerLane) {
        set_error("rmu_debug_layernorm: hidden must be a multiple of 128, at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_layernorm(pre, T, H, gamma, beta, eps, reinterpret_cast<__half*>(out_hi), reinterpret_cast<__half*>(out_lo),
                            static_cast<cudaStream_t>(stream));
}

int rmu_debug_embed_ln(const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T, int H, int vocab,
                       int max_pos, int type_vocab, const float* word, const float* pos, const float* typ,
                       const float* gamma, const float* beta, float eps, uint16_t* out_hi, uint16_t* out_lo, void* stream) {
    if (!ids || !cu || !word || !pos || !typ || !gamma || !beta || !out_hi || !out_lo || B <= 0 || T <= 0 || H <= 0 ||
        vocab <= 0 || max_pos <= 0 || type_vocab <= 0) {
        set_error("rmu_debug_embed_ln: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % 128 != 0 || H > 32 * kMaxPerLane) {
        set_error("rmu_debug_embed_ln: hidden must be a multiple of 128, at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_embed_ln(ids, type_ids, cu, B, T, H, vocab, max_pos, type_vocab, word, pos, typ, gamma, beta, eps,
                           reinterpret_cast<__half*>(out_hi), reinterpret_cast<__half*>(out_lo), static_cast<cudaStream_t>(stream));
}

int rmu_debug_embed_ln_pos(const int32_t* ids, const int32_t* type_ids, const int32_t* cu, int B, int T, int H, int vocab,
                           int max_pos, int type_vocab, const float* word, const float* pos, const float* typ,
                           const float* gamma, const float* beta, float eps, int pos_mode, uint16_t* out_hi,
                           uint16_t* out_lo, void* stream) {
    if (pos_mode != RMU_POS_ABSOLUTE && pos_mode != RMU_POS_OFFSET) {
        set_error("rmu_debug_embed_ln_pos: pos_mode must be RMU_POS_ABSOLUTE or RMU_POS_OFFSET");
        return RMU_ERR_ARG;
    }
    if (!ids || !cu || !word || !pos || !typ || !gamma || !beta || !out_hi || !out_lo || B <= 0 || T <= 0 || H <= 0 ||
        vocab <= 0 || max_pos <= 0 || type_vocab <= 0) {
        set_error("rmu_debug_embed_ln_pos: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % 128 != 0 || H > 32 * kMaxPerLane) {
        set_error("rmu_debug_embed_ln_pos: hidden must be a multiple of 128, at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_embed_ln(ids, type_ids, cu, B, T, H, vocab, max_pos, type_vocab, word, pos, typ, gamma, beta, eps,
                           reinterpret_cast<__half*>(out_hi), reinterpret_cast<__half*>(out_lo), static_cast<cudaStream_t>(stream),
                           pos_mode);
}

int rmu_relative_bias_table(const float* bias_h, int buckets, int heads, float* table_h) {
    if (!bias_h || !table_h || heads <= 0) { set_error("rmu_relative_bias_table: bad argument"); return RMU_ERR_ARG; }
    if (buckets != 32) { set_error("rmu_relative_bias_table: buckets must be 32"); return RMU_ERR_UNSUPPORTED; }
    build_relative_bias_table(bias_h, heads, table_h);
    return RMU_OK;
}

int rmu_debug_attention_bias(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const uint16_t* cls_q_hi, const uint16_t* cls_q_lo,
                             const int32_t* cu, int B, int H, int heads, int max_seqlen, const float* rel_table,
                             uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !rel_table || !ctx_hi || !ctx_lo || (!cls_q_hi) != (!cls_q_lo) || B <= 0 ||
        heads <= 0 || H <= 0 || max_seqlen <= 0) {
        set_error("rmu_debug_attention_bias: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % heads != 0 || (H / heads != 32 && H / heads != 64)) {
        set_error("rmu_debug_attention_bias: head_dim must be 32 or 64");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_attention(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo),
                            reinterpret_cast<const __half*>(cls_q_hi), reinterpret_cast<const __half*>(cls_q_lo), cu, B, H,
                            heads, max_seqlen, reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo),
                            static_cast<cudaStream_t>(stream), rel_table);
}

int rmu_log_bucket_table(int buckets, int max_position, int n, int32_t* out_h) {
    if (!out_h || n < 1) { set_error("rmu_log_bucket_table: bad argument"); return RMU_ERR_ARG; }
    if (buckets < 2 || max_position < buckets / 2 + 2) {
        set_error("rmu_log_bucket_table: buckets must be at least 2 and max_position at least buckets / 2 + 2");
        return RMU_ERR_UNSUPPORTED;
    }
    for (int r = -(n - 1); r <= n - 1; ++r) out_h[r + n - 1] = log_bucket(r, buckets, max_position);
    return RMU_OK;
}

int rmu_debug_attention_disentangled(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const uint16_t* cls_q_hi,
                                     const uint16_t* cls_q_lo, const int32_t* cu, int B, int T, int H, int heads,
                                     int max_seqlen, const uint16_t* pos_hi, const uint16_t* pos_lo, int position_buckets,
                                     const int32_t* cidx_h, float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo,
                                     void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !pos_hi || !pos_lo || !cidx_h || !ws || !ctx_hi || !ctx_lo ||
        (!cls_q_hi) != (!cls_q_lo) || B <= 0 || T <= 0 || heads <= 0 || H <= 0 || max_seqlen <= 0 || ws_elems < 0 ||
        position_buckets <= 0) {
        set_error("rmu_debug_attention_disentangled: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % heads != 0 || H / heads != 64) {
        set_error("rmu_debug_attention_disentangled: head_dim must be 64");
        return RMU_ERR_ARG;
    }
    const int rmax = max_seqlen - 1;
    // P1 reads rows cidx_h[0] .. cidx_h[2 rmax] of the pos planes, which hold 2 position_buckets rows
    for (int k = 0; k < 2 * rmax; ++k)
        if (cidx_h[k + 1] < cidx_h[k] || cidx_h[k] < 0) {
            set_error("rmu_debug_attention_disentangled: cidx must be non-negative and non-decreasing");
            return RMU_ERR_ARG;
        }
    if (cidx_h[2 * rmax] >= 2 * position_buckets) {
        set_error("rmu_debug_attention_disentangled: cidx reaches past the 2 * position_buckets rows of the pos planes");
        return RMU_ERR_ARG;
    }
    const bool cls = cls_q_hi != nullptr;
    const size_t terms = position_ws_floats(cidx_h, rmax, max_seqlen, cls ? B : T, T, heads);
    if (static_cast<size_t>(ws_elems) < terms + 2 * static_cast<size_t>(rmax) + 1) {
        set_error("rmu_debug_attention_disentangled: workspace too small");
        return RMU_ERR_ARG;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int* cidx_d = reinterpret_cast<int*>(ws + terms);
    RMU_CUDA(cudaMemcpyAsync(cidx_d, cidx_h, (2 * static_cast<size_t>(rmax) + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    return run_disentangled_attention(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo),
                                      reinterpret_cast<const __half*>(cls_q_hi), reinterpret_cast<const __half*>(cls_q_lo), cu,
                                      B, T, H, heads, max_seqlen, reinterpret_cast<const __half*>(pos_hi),
                                      reinterpret_cast<const __half*>(pos_lo), cidx_d, cidx_h, rmax, ws,
                                      reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo), st);
}

int rmu_debug_pool(const uint16_t* hi, const uint16_t* lo, const int32_t* cu, int B, int H, int pool_mode, int normalize,
                   float* out, void* stream) {
    if (!hi || !lo || !cu || !out || B <= 0 || H <= 0 || (pool_mode != RMU_POOL_MEAN && pool_mode != RMU_POOL_CLS)) {
        set_error("rmu_debug_pool: bad argument");
        return RMU_ERR_ARG;
    }
    if (H > 1024) {
        set_error("rmu_debug_pool: hidden must be at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_pool(reinterpret_cast<const __half*>(hi), reinterpret_cast<const __half*>(lo), cu, B, H, pool_mode, normalize,
                       false, out, static_cast<cudaStream_t>(stream));
}

int rmu_debug_cls_head(const uint16_t* hi, const uint16_t* lo, const int32_t* cu, int B, int H, int num_labels,
                       const float* pw, const float* pb, const float* cw, const float* cb, float* out, void* stream) {
    if (!hi || !lo || !cu || !pw || !pb || !cw || !cb || !out || B <= 0 || H <= 0 || num_labels <= 0) {
        set_error("rmu_debug_cls_head: bad argument");
        return RMU_ERR_ARG;
    }
    if (H > 1024) {
        set_error("rmu_debug_cls_head: hidden must be at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_cls_head(reinterpret_cast<const __half*>(hi), reinterpret_cast<const __half*>(lo), cu, B, H, num_labels,
                           false, pw, pb, cw, cb, out, static_cast<cudaStream_t>(stream));
}

int rmu_debug_encoder_position_planes(const rmu_encoder* e, int layer, uint16_t* hi, uint16_t* lo, void* stream) {
    if (!e || !hi || !lo || e->ext.position_buckets <= 0 || layer < 0 || layer >= e->cfg.layers) {
        set_error("rmu_debug_encoder_position_planes: bad argument (an encoder with position_buckets > 0 and a layer of it)");
        return RMU_ERR_ARG;
    }
    const EncLayer& L = e->layers[layer];
    const size_t n = static_cast<size_t>(2) * e->ext.position_buckets * 2 * e->cfg.hidden * sizeof(__half);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RMU_CUDA(cudaMemcpyAsync(hi, L.pos_hi, n, cudaMemcpyDeviceToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(lo, L.pos_lo, n, cudaMemcpyDeviceToDevice, st));
    return RMU_OK;
}

int rmu_debug_cls_head_act(const uint16_t* hi, const uint16_t* lo, const int32_t* cu, int B, int H, int num_labels,
                           const float* pw, const float* pb, const float* cw, const float* cb, int head_act, float* out,
                           void* stream) {
    if (!hi || !lo || !cu || !pw || !pb || !cw || !cb || !out || B <= 0 || H <= 0 || num_labels <= 0 ||
        (head_act != RMU_HEAD_TANH && head_act != RMU_HEAD_GELU && head_act != RMU_HEAD_RELU)) {
        set_error("rmu_debug_cls_head_act: bad argument");
        return RMU_ERR_ARG;
    }
    if (H > 1024) {
        set_error("rmu_debug_cls_head_act: hidden must be at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_cls_head(reinterpret_cast<const __half*>(hi), reinterpret_cast<const __half*>(lo), cu, B, H, num_labels,
                           false, pw, pb, cw, cb, out, static_cast<cudaStream_t>(stream), head_act);
}

int rmu_debug_dense(const float* x, int B, int n_in, int n_out, const float* W, const float* b, int act, int normalize,
                    float* y, void* stream) {
    if (!x || !W || !y || B <= 0 || n_in <= 0 || n_out <= 0) { set_error("rmu_debug_dense: bad argument"); return RMU_ERR_ARG; }
    if (act != RMU_DENSE_IDENTITY && act != RMU_DENSE_TANH) {
        set_error("rmu_debug_dense: act must be RMU_DENSE_IDENTITY (0) or RMU_DENSE_TANH (1)");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_dense(x, B, n_in, n_out, W, b, act, normalize, y, static_cast<cudaStream_t>(stream));
}

int rmu_debug_attention_window(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, int B, int H, int heads,
                               int max_seqlen, int window, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !ctx_hi || !ctx_lo || B <= 0 || heads <= 0 || H <= 0 || max_seqlen <= 0 || window <= 0) {
        set_error("rmu_debug_attention_window: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % heads != 0 || (H / heads != 32 && H / heads != 64)) {
        set_error("rmu_debug_attention_window: head_dim must be 32 or 64");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_attention(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), nullptr, nullptr,
                            cu, B, H, heads, max_seqlen, reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo),
                            static_cast<cudaStream_t>(stream), nullptr, nullptr, nullptr, window);
}

int rmu_debug_modernbert_head(const float* pooled, int B, int H, int num_labels, const float* dense_w, const float* dense_b,
                              const float* norm_w, const float* norm_b, float eps, const float* cw, const float* cb,
                              float* out, void* stream) {
    if (!pooled || !dense_w || !dense_b || !norm_w || !norm_b || !cw || !cb || !out || B <= 0 || H <= 0 || num_labels <= 0) {
        set_error("rmu_debug_modernbert_head: bad argument");
        return RMU_ERR_ARG;
    }
    if (H > 1024) {
        set_error("rmu_debug_modernbert_head: hidden must be at most 1024");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_mb_head(pooled, B, H, num_labels, dense_w, dense_b, norm_w, norm_b, eps, cw, cb, out,
                          static_cast<cudaStream_t>(stream));
}

int rmu_debug_rmsnorm(const float* x, int T, int H, const float* w, float eps, uint16_t* hi, uint16_t* lo,
                      int32_t* range_flag, void* stream) {
    if (!x || !w || !hi || !lo || T <= 0 || H <= 0) { set_error("rmu_debug_rmsnorm: bad argument"); return RMU_ERR_ARG; }
    if (H % 128 != 0 || H > kRmsMaxHidden) { set_error("rmu_debug_rmsnorm: H must be a multiple of 128 up to 8192"); return RMU_ERR_UNSUPPORTED; }
    return launch_rms_split(x, T, H, w, eps, reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo), range_flag,
                            static_cast<cudaStream_t>(stream));
}

int rmu_debug_qk_norm_rope(const float* qkv, int T, int heads, int kv_heads, const int32_t* pos, const float* q_norm,
                           const float* k_norm, float eps, float qscale, const float* rope_cos, const float* rope_sin,
                           int rope_rows, uint16_t* hi, uint16_t* lo, int32_t* range_flag, void* stream) {
    // both norms null: Llama's step without the per-head RMSNorm; exactly one null is a caller error
    if (!qkv || !pos || !q_norm != !k_norm || !rope_cos || !rope_sin || !hi || !lo || T <= 0 || heads <= 0 ||
        kv_heads <= 0 || rope_rows <= 0) {
        set_error("rmu_debug_qk_norm_rope: bad argument");
        return RMU_ERR_ARG;
    }
    return launch_qk_norm_rope(qkv, T, heads, kv_heads, pos, q_norm, k_norm, eps, qscale, rope_cos, rope_sin, rope_rows,
                               reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo), range_flag,
                               static_cast<cudaStream_t>(stream));
}

int rmu_debug_attention_causal(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, int B, int heads,
                               int kv_heads, int max_seqlen, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    if (!qkv_hi || !qkv_lo || !cu || !ctx_hi || !ctx_lo || B <= 0 || heads <= 0 || kv_heads <= 0 || max_seqlen <= 0) {
        set_error("rmu_debug_attention_causal: bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) {
        set_error("rmu_debug_attention_causal: heads must be a multiple of kv_heads");
        return RMU_ERR_UNSUPPORTED;
    }
    return launch_attention_causal(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), cu, B,
                                   heads, kv_heads, max_seqlen, reinterpret_cast<__half*>(ctx_hi),
                                   reinterpret_cast<__half*>(ctx_lo), static_cast<cudaStream_t>(stream));
}

int rmu_debug_attention_spans(const uint16_t* qkv_hi, const uint16_t* qkv_lo, int T, int heads, int kv_heads,
                              const int32_t* spans, int n_spans, double* out, void* stream) {
    if (!qkv_hi || !qkv_lo || !spans || !out || T <= 0 || heads <= 0 || kv_heads <= 0 || n_spans <= 0) {
        set_error("rmu_debug_attention_spans: bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) {
        set_error("rmu_debug_attention_spans: heads must be a multiple of kv_heads");
        return RMU_ERR_UNSUPPORTED;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* ws = nullptr;
    RMU_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&ws), attention_spans_ws_floats(T, heads) * sizeof(float), st));
    const int rc = launch_attention_spans(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), T,
                                          heads, kv_heads, spans, n_spans, ws, out, st);
    RMU_CUDA(cudaFreeAsync(ws, st));
    return rc;
}

int rmu_debug_last_token(const float* x, const int32_t* ids, const int32_t* cu, int B, int H, const float* w, float eps,
                         int pad_id, int normalize, const float* head, int num_labels, float* out, void* stream) {
    if (!x || !ids || !cu || !w || !out || B <= 0 || H <= 0 || (head && num_labels <= 0)) {
        set_error("rmu_debug_last_token: bad argument");
        return RMU_ERR_ARG;
    }
    if (H % 128 != 0 || H > 4096) { set_error("rmu_debug_last_token: H must be a multiple of 128 up to 4096"); return RMU_ERR_UNSUPPORTED; }
    return launch_last_token(x, ids, cu, B, H, w, eps, pad_id, normalize, head, num_labels, out, static_cast<cudaStream_t>(stream));
}

int rmu_debug_split_planes(const float* src, int64_t n, uint16_t* hi, uint16_t* lo, void* stream) {
    if (!src || !hi || !lo || n < 0) {
        set_error("rmu_debug_split_planes: bad argument");
        return RMU_ERR_ARG;
    }
    return launch_split_planes(src, static_cast<size_t>(n), reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo),
                               static_cast<cudaStream_t>(stream));
}

int rmu_debug_join_planes(const uint16_t* hi, const uint16_t* lo, int64_t n, float* out, void* stream) {
    if (!hi || !lo || !out || n < 0) {
        set_error("rmu_debug_join_planes: bad argument");
        return RMU_ERR_ARG;
    }
    return launch_join_planes(reinterpret_cast<const __half*>(hi), reinterpret_cast<const __half*>(lo), static_cast<size_t>(n),
                              out, static_cast<cudaStream_t>(stream));
}


int rmu_debug_attention_decode(const uint16_t* q_hi, const uint16_t* q_lo, const uint16_t* kv, int heads, int kv_heads,
                               int cap, int n, float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo,
                               void* stream) {
    if (!q_hi || !q_lo || !kv || !ws || !ctx_hi || !ctx_lo || heads < 1 || kv_heads < 1 || n < 1 || cap < n) {
        set_error("rmu_debug_attention_decode: bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) { set_error("rmu_debug_attention_decode: heads % kv_heads != 0"); return RMU_ERR_UNSUPPORTED; }
    if (ws_elems < 0 || static_cast<size_t>(ws_elems) < decode_part_floats(heads, n)) {
        set_error("rmu_debug_attention_decode: the workspace needs " + std::to_string(decode_part_floats(heads, n)) + " floats");
        return RMU_ERR_ARG;
    }
    return launch_attention_decode(reinterpret_cast<const __half*>(q_hi), reinterpret_cast<const __half*>(q_lo),
                                   reinterpret_cast<const __half*>(kv), heads, kv_heads, cap, n, ws,
                                   reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo),
                                   static_cast<cudaStream_t>(stream));
}

int rmu_debug_attention_decode_rows(const uint16_t* q_hi, const uint16_t* q_lo, int64_t qld, int B, const uint16_t* kv,
                                    int heads, int kv_heads, int cap, int P, const int32_t* pos_h, const int32_t* shift_h,
                                    float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    const std::string fn("rmu_debug_attention_decode_rows");
    if (!q_hi || !q_lo || !kv || !pos_h || !shift_h || !ws || !ctx_hi || !ctx_lo || B < 1 || B > 65535 || heads < 1 ||
        kv_heads < 1 || P < 0 || qld < static_cast<int64_t>(heads) * kQwenHD) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) { set_error(fn + ": heads % kv_heads != 0"); return RMU_ERR_UNSUPPORTED; }
    int n = 1;
    for (int b = 0; b < B; ++b) {
        // every key the row reads lies in [0, cap): the prefix rows and its own rows pos + shift
        if (pos_h[b] < 0 || shift_h[b] < 0 || std::min(pos_h[b] + 1, P) > cap ||
            (pos_h[b] >= P && static_cast<int64_t>(pos_h[b]) + shift_h[b] >= cap)) {
            set_error(fn + ": row " + std::to_string(b) + " reads past the cache");
            return RMU_ERR_ARG;
        }
        n = std::max(n, pos_h[b] + 1);
    }
    const size_t part = static_cast<size_t>(B) * decode_part_floats(heads, n);
    if (ws_elems < 0 || static_cast<size_t>(ws_elems) < part + 2 * static_cast<size_t>(B)) {
        set_error(fn + ": the workspace needs " + std::to_string(part + 2 * static_cast<size_t>(B)) + " floats");
        return RMU_ERR_ARG;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int* rows = reinterpret_cast<int*>(ws + part);
    RMU_CUDA(cudaMemcpyAsync(rows, pos_h, static_cast<size_t>(B) * sizeof(int), cudaMemcpyHostToDevice, st));
    RMU_CUDA(cudaMemcpyAsync(rows + B, shift_h, static_cast<size_t>(B) * sizeof(int), cudaMemcpyHostToDevice, st));
    DecRows dr;
    dr.pos = rows;
    dr.shift = rows + B;
    dr.P = P;
    dr.qld = static_cast<size_t>(qld);
    return launch_attention_decode(reinterpret_cast<const __half*>(q_hi), reinterpret_cast<const __half*>(q_lo),
                                   reinterpret_cast<const __half*>(kv), heads, kv_heads, cap, n, ws,
                                   reinterpret_cast<__half*>(ctx_hi), reinterpret_cast<__half*>(ctx_lo), st, B, dr);
}

int rmu_debug_attention_cached(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, int B, int heads,
                               int kv_heads, const uint16_t* kv, int cap, int P, const int32_t* shift, int max_own,
                               uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream) {
    const std::string fn("rmu_debug_attention_cached");
    if (!qkv_hi || !qkv_lo || !cu || !kv || !shift || !ctx_hi || !ctx_lo || B < 1 || B > kMaxGridY || heads < 1 ||
        kv_heads < 1 || P < 0 || max_own < 1 || cap < P) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) { set_error(fn + ": heads must be a multiple of kv_heads"); return RMU_ERR_UNSUPPORTED; }
    PrefixKeys pk;
    pk.kv = reinterpret_cast<const __half*>(kv);
    pk.shift = shift;
    pk.cap = cap;
    pk.P = P;
    return launch_attention_cached(reinterpret_cast<const __half*>(qkv_hi), reinterpret_cast<const __half*>(qkv_lo), cu, B,
                                   heads, kv_heads, max_own, pk, reinterpret_cast<__half*>(ctx_hi),
                                   reinterpret_cast<__half*>(ctx_lo), static_cast<cudaStream_t>(stream));
}

int rmu_debug_kv_append(const uint16_t* hi, const uint16_t* lo, int T, int heads, int kv_heads, int pos0, int cap,
                        uint16_t* kv, void* stream) {
    if (!hi || !lo || !kv || T < 1 || heads < 1 || kv_heads < 1 || pos0 < 0 ||
        static_cast<int64_t>(pos0) + T > cap) {
        set_error("rmu_debug_kv_append: bad argument");
        return RMU_ERR_ARG;
    }
    if (heads % kv_heads != 0) { set_error("rmu_debug_kv_append: heads % kv_heads != 0"); return RMU_ERR_UNSUPPORTED; }
    return launch_kv_append(reinterpret_cast<const __half*>(hi), reinterpret_cast<const __half*>(lo), T, heads, kv_heads,
                            pos0, cap, reinterpret_cast<__half*>(kv), static_cast<cudaStream_t>(stream));
}

int rmu_debug_nf4_quantize(const uint16_t* hi, int64_t n, uint8_t* codes, float* absmax, void* stream) {
    if (!hi || !codes || !absmax || n < 1) { set_error("rmu_debug_nf4_quantize: bad argument"); return RMU_ERR_ARG; }
    if (n % kNf4Block != 0) { set_error("rmu_debug_nf4_quantize: n % 64 != 0"); return RMU_ERR_UNSUPPORTED; }
    return launch_nf4_quantize(reinterpret_cast<const __half*>(hi), n, codes, absmax, static_cast<cudaStream_t>(stream));
}

int rmu_debug_nf4_dequantize(const uint8_t* codes, const float* absmax, int64_t n, uint16_t* hi, void* stream) {
    if (!codes || !absmax || !hi || n < 1) { set_error("rmu_debug_nf4_dequantize: bad argument"); return RMU_ERR_ARG; }
    if (n % kNf4Block != 0) { set_error("rmu_debug_nf4_dequantize: n % 64 != 0"); return RMU_ERR_UNSUPPORTED; }
    return launch_nf4_dequantize(codes, absmax, n, reinterpret_cast<__half*>(hi), static_cast<cudaStream_t>(stream));
}

int rmu_debug_nf4_gemv(int mode, const uint16_t* x_hi, const uint16_t* x_lo, const uint8_t* codes, const float* absmax,
                       int N, int K, const float* bias, const float* res_f32, float* out_f32, uint16_t* out_hi,
                       uint16_t* out_lo, int32_t* range_flag, void* stream) {
    const std::string fn("rmu_debug_nf4_gemv");
    if (mode != GEMM_BIAS_F32 && mode != GEMM_BIAS_RESF32_F32 && mode != GEMM_BIAS_SWIGLU_SPLIT) {
        set_error(fn + ": mode must be 0, 6 or 7");
        return RMU_ERR_ARG;
    }
    const bool swiglu = mode == GEMM_BIAS_SWIGLU_SPLIT;
    if (!x_hi || !x_lo || !codes || !absmax || !bias || N < 1 || K < 1 || (swiglu ? !out_hi || !out_lo : !out_f32) ||
        (mode == GEMM_BIAS_RESF32_F32 && !res_f32)) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    if (N % 128 != 0 || K % kNf4Block != 0 || K > kNf4MaxK) {
        set_error(fn + ": N must be a multiple of 128 and K a multiple of 64 up to " + std::to_string(kNf4MaxK));
        return RMU_ERR_UNSUPPORTED;
    }
    GemmParams p{};
    p.M = 1; p.N = N; p.K = K; p.bias = bias; p.out_f32 = out_f32; p.res_f32 = res_f32;
    p.out_hi = reinterpret_cast<__half*>(out_hi); p.out_lo = reinterpret_cast<__half*>(out_lo);
    p.range_flag = reinterpret_cast<int*>(range_flag);
    Nf4Weight W;
    W.codes = const_cast<uint8_t*>(codes); W.absmax = const_cast<float*>(absmax); W.rows = N; W.cols = K;
    return launch_nf4_gemv(mode, reinterpret_cast<const __half*>(x_hi), reinterpret_cast<const __half*>(x_lo), W, p,
                           device_sm_count(), static_cast<cudaStream_t>(stream));
}

int rmu_debug_nf4_gemv_rows(int mode, int M, const uint16_t* x_hi, const uint16_t* x_lo, const uint8_t* codes,
                            const float* absmax, int N, int K, const float* bias, const float* res_f32, float* out_f32,
                            uint16_t* out_hi, uint16_t* out_lo, int32_t* range_flag, void* stream) {
    const std::string fn("rmu_debug_nf4_gemv_rows");
    if (mode != GEMM_BIAS_F32 && mode != GEMM_BIAS_RESF32_F32 && mode != GEMM_BIAS_SWIGLU_SPLIT) {
        set_error(fn + ": mode must be 0, 6 or 7");
        return RMU_ERR_ARG;
    }
    const bool swiglu = mode == GEMM_BIAS_SWIGLU_SPLIT;
    if (!x_hi || !x_lo || !codes || !absmax || !bias || M < 1 || M > kNf4MaxRows || N < 1 || K < 1 ||
        (swiglu ? !out_hi || !out_lo : !out_f32) || (mode == GEMM_BIAS_RESF32_F32 && !res_f32)) {
        set_error(fn + ": bad argument (M must be 1 .. " + std::to_string(kNf4MaxRows) + ")");
        return RMU_ERR_ARG;
    }
    if (N % 128 != 0 || K % kNf4Block != 0 || K > kNf4MaxK) {
        set_error(fn + ": N must be a multiple of 128 and K a multiple of 64 up to " + std::to_string(kNf4MaxK));
        return RMU_ERR_UNSUPPORTED;
    }
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.bias = bias; p.out_f32 = out_f32; p.res_f32 = res_f32;
    p.out_hi = reinterpret_cast<__half*>(out_hi); p.out_lo = reinterpret_cast<__half*>(out_lo);
    p.range_flag = reinterpret_cast<int*>(range_flag);
    Nf4Weight W;
    W.codes = const_cast<uint8_t*>(codes); W.absmax = const_cast<float*>(absmax); W.rows = N; W.cols = K;
    return launch_nf4_gemv_rows(mode, reinterpret_cast<const __half*>(x_hi), reinterpret_cast<const __half*>(x_lo), W, p,
                                device_sm_count(), static_cast<cudaStream_t>(stream));
}

int rmu_debug_nf4_conversion(const rmu_encoder* e, int64_t* peak, int64_t* delta) {
    if (!e || !peak || !delta) { set_error("rmu_debug_nf4_conversion: bad argument"); return RMU_ERR_ARG; }
    if (!e->nf4) { set_error("rmu_debug_nf4_conversion: the handle's weights are not NF4"); return RMU_ERR_ARG; }
    *peak = e->nf4_peak;
    *delta = e->nf4_delta;
    return RMU_OK;
}

int rmu_debug_sample(float* logits, int V, uint32_t* presence, const rmu_sampling* s, float u, int32_t* token,
                     void* stream) {
    if (!logits || V < 1 || !presence || !s || !token || !(u >= 0.f && u < 1.f)) {
        set_error("rmu_debug_sample: bad argument");
        return RMU_ERR_ARG;
    }
    const int rc = check_sampling("rmu_debug_sample", s);
    if (rc != RMU_OK) return rc;
    const SampleArgs sa = sample_args(*s);
    return launch_sample(logits, V, presence, sa, u, 0ull, 0ull, token, static_cast<cudaStream_t>(stream));
}

int rmu_debug_sample_rows(float* logits, int V, int B, uint32_t* presence, const int32_t* seq, const uint64_t* seeds,
                          int64_t step, const rmu_sampling* s, int32_t* token, void* stream) {
    if (!logits || V < 1 || B < 1 || !presence || !seq || !seeds || !s || !token || step < 0) {
        set_error("rmu_debug_sample_rows: bad argument");
        return RMU_ERR_ARG;
    }
    const int rc = check_sampling("rmu_debug_sample_rows", s);
    if (rc != RMU_OK) return rc;
    const SampleArgs sa = sample_args(*s);
    SampleRows sr;
    sr.seq = seq;
    sr.seeds = reinterpret_cast<const unsigned long long*>(seeds);
    sr.words = (static_cast<size_t>(V) + 31) / 32;
    return launch_sample(logits, V, presence, sa, -1.f, 0ull, static_cast<unsigned long long>(step), token,
                         static_cast<cudaStream_t>(stream), B, sr);
}

int rmu_debug_sample_verify_rows(float* logits, int V, int M, uint32_t* presence, const int32_t* ids, uint64_t seed,
                                 int64_t step0, const rmu_sampling* s, uint32_t* rows, int32_t* token, void* stream) {
    if (!logits || V < 1 || M < 1 || M > RMU_MAX_GENERATE_BATCH || !presence || !ids || !s || !rows || !token || step0 < 0) {
        set_error("rmu_debug_sample_verify_rows: bad argument");
        return RMU_ERR_ARG;
    }
    int rc = check_sampling("rmu_debug_sample_verify_rows", s);
    if (rc != RMU_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const SampleArgs sa = sample_args(*s);
    SampleRows sr;
    sr.words = (static_cast<size_t>(V) + 31) / 32;
    sr.row_step = true;
    rc = launch_presence_rows(presence, sr.words, ids, M, rows, st);
    if (rc != RMU_OK) return rc;
    return launch_sample(logits, V, rows, sa, -1.f, seed, static_cast<unsigned long long>(step0), token, st, M, sr);
}

int rmu_debug_sample_session_rows(float* logits, int V, int B, uint32_t* presence, const int32_t* seq,
                                  const uint64_t* seeds, const uint64_t* steps, int n_seq, const rmu_sampling* s_h,
                                  int32_t* token, void* stream) {
    const std::string fn("rmu_debug_sample_session_rows");
    if (!logits || V < 1 || B < 1 || !presence || !seq || !seeds || !steps || n_seq < 1 ||
        n_seq > RMU_MAX_GENERATE_BATCH || !s_h || !token) {
        set_error(fn + ": bad argument");
        return RMU_ERR_ARG;
    }
    SampleArgs sa[RMU_MAX_GENERATE_BATCH];
    for (int q = 0; q < n_seq; ++q) {
        const int rc = check_sampling(fn, s_h + q);
        if (rc != RMU_OK) return rc;
        sa[q] = sample_args(s_h[q]);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SampleArgs* d_args = nullptr;
    RMU_CUDA(cudaMalloc(&d_args, sizeof(sa)));
    int rc = RMU_OK;
    if (cudaMemcpyAsync(d_args, sa, sizeof(sa), cudaMemcpyHostToDevice, st) != cudaSuccess) {
        set_error(fn + ": cannot upload the settings");
        rc = RMU_ERR_CUDA;
    }
    SampleRows sr;
    sr.seq = seq;
    sr.seeds = reinterpret_cast<const unsigned long long*>(seeds);
    sr.words = (static_cast<size_t>(V) + 31) / 32;
    sr.args = d_args;
    sr.steps = reinterpret_cast<const unsigned long long*>(steps);
    if (rc == RMU_OK) rc = launch_sample(logits, V, presence, SampleArgs{}, -1.f, 0ull, 0ull, token, st, B, sr);
    if (cudaStreamSynchronize(st) != cudaSuccess && rc == RMU_OK) { set_error(fn + ": stream failed"); rc = RMU_ERR_CUDA; }
    cudaFree(d_args);
    return rc;
}

}  // extern "C"
