// Coarse top-k scan of the flat index (sm_90a) and its selection kernel.  Included by rmu_index.cu inside
// namespace rmu, after block_sum / warp_bitonic_desc / block_radix_select and the top-k tail (block_collect,
// block_sort_desc, write_topk).
//
// Stands behind the reference's brute-force search (col.search of the retriever built at
// server/RAGHelper.py:497-499; Milvus-lite FLAT / pgvector sequential scan on the CPU).
//
// Geometry.  The fp32 corpus streams HBM -> smem through TMA exactly once as 16 KB boxes (128 rows x 32
// floats, SWIZZLE_128B) and is consumed in place as the **A operand** of wgmma tf32: each of the two consumer
// warpgroups takes 64 rows of a 128-row tile (M = 64), the queries are the B operand (N = NQ <= 64 per launch),
// resident in shared memory for the whole launch ([K block][NQ rows x 128 B], loaded once by TMA, zero filled past
// nq / dim, padded to whole pipeline stages).  Whatever shared memory the query block leaves is the ring of corpus
// boxes in flight.
// The accumulator D[64 rows x NQ queries] lives in the registers of the warpgroup (NQ / 2 per thread).  The slot of a
// K stage is handed back to the TMA warp as soon as its MMAs have retired, so the producer keeps streaming the next
// tile while the consumers run the epilogue of this one.
//
// Epilogue: every accumulator element (corpus row, query) is compared with the query's running threshold tau;
// the few that pass are appended (shared-memory counter, global list) to the (CTA, query) candidate list.  At tile
// boundaries lists past 95 entries are sorted by one warp each (warp-shuffle bitonic network) and cut to their best
// 64; the 64th key becomes the list's floor.
// Threshold exchange without a second launch: whenever a list is sorted, its 16th best key is published with an
// atomicMax into gmax[query][cta % groups].  If every one of `groups` disjoint groups of CTAs contains a
// CTA with >= 16 keys >= v, then >= 16 * groups rows score >= v: tau = min over groups of the group maxima is
// a valid lower bound of the (16 * groups)-th best key of the whole corpus.  groups = KSEL / 16, so nothing that
// belongs to the global best KSEL is ever rejected (ties at tau are covered by the certificate's bound).
// gmax entries are tagged with a per-search epoch in their high word, so they never need clearing.
#pragma once

constexpr int kTileRows = 128;                   // corpus rows per CTA tile (two warpgroups x M = 64)
constexpr int kBoxBytes = kTileRows * 128;       // one TMA box: 128 rows x 32 fp32
constexpr int kScanConsumerWarps = 8;            // two warpgroups: MMA + epilogue
constexpr int kScanThreads = 32 * kScanConsumerWarps + 32;   // + TMA producer warp
constexpr int kListCap = 256;                    // slots of a (CTA, query) candidate list
constexpr int kListKeep = 64;                    // entries a list keeps when it is sorted and cut
constexpr int kListTrig = 95;                    // a list longer than this at a tile boundary is sorted and cut
                                                 // (one tile adds <= 128 entries to a list: 95 + 128 < kListCap)
constexpr int kPubRank = 16;                     // the published key of a list: its 16th best
constexpr int kGroupsMax = 16;                   // gmax row length; KSEL <= 16 * kPubRank = 256
constexpr int kScanStateBytes = 2048;            // mbarriers + per-query state behind the ring
constexpr int kScanQOpMax = 96 * 1024;           // shared memory the resident query operand may take
constexpr int kScanKD = 2;                       // boxes (128-byte K blocks) per pipeline stage
constexpr int kScanMaxStages = 16;
constexpr int kScanMaxQ = 64;                    // queries per launch (MMA N)

struct ScanParams {
    int nq;                    // live queries of this launch (<= NQ); query j = row j of tmap_q
    int dim;
    long long n;               // rows in the index
    int ntiles;                // ceil(n / 128)
    int nstages;               // ring depth, in stages of KD boxes
    int metric;
    const float* rscale;       // [n] 1/||x|| (cosine), used unless the corpus is unit-norm
    const float* rbias;        // [n] -0.5 ||x||^2 (L2), used unless the corpus is unit-norm
    const unsigned* stats_bits;   // [1] = max over rows of | ||x||^2 - 1 | (float bits): < 1e-6 => unit rows
    unsigned long long* lists; // [grid][NQ][kListCap]
    int* counts;               // [grid][NQ] entries valid in each list when the launch ends
    float* floors;             // [grid][NQ] largest score the list ever cut away (-inf: never cut)
    unsigned long long* gmax;  // [NQ][kGroupsMax]  (epoch << 32 | ordered score), see above
    unsigned epoch;
    int groups;                // 0: no exchange (grids smaller than the group count)
    float* dbg;                // diagnostics: raw accumulators of the first 256 rows, [NQ][256]
    // second pass for queries whose certificate failed ("pool mode", fixed_tau != nullptr): every row whose coarse key
    // beats the query's FIXED threshold is appended to a per-query pool; no lists, no exchange
    const float* fixed_tau;    // [NQ] thresholds of the launch's query slots
    unsigned long long* pool;  // [NQ][pool_cap]
    int* pool_cnt;             // [NQ] entries appended (may exceed pool_cap: overflow, the query stays flagged)
    int pool_cap;
    const int* nq_dev;         // nullable: live queries of the pass (device count of flagged queries)
    int q_off;                 // this launch serves slots q_off .. q_off + nq - 1 of them
};

// sort one candidate list (n <= 32 * E entries) descending, keep its best kListKeep, publish its kPubRank-th key
template <int E>
__device__ __forceinline__ void scan_sort_list(unsigned long long* b, int n, int& cnt, float& floor_v,
                                               unsigned long long* gslot, unsigned epoch) {
    const unsigned lane = lane_id();
    unsigned long long v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int i = e * 32 + static_cast<int>(lane);
        v[e] = (i < n) ? b[i] : 0ull;
    }
    warp_bitonic_desc<E>(v);
    b[lane] = v[0];
    b[32 + lane] = v[1];
    const unsigned long long k_pub = __shfl_sync(0xffffffffu, v[0], kPubRank - 1);
    const unsigned long long k_keep = __shfl_sync(0xffffffffu, v[1], 31);
    if (lane == 0) {
        if (n > kListKeep) { cnt = kListKeep; floor_v = fmaxf(floor_v, key_score(k_keep)); }
        if (n >= kPubRank && gslot != nullptr)
            atomicMax(gslot, (static_cast<unsigned long long>(epoch) << 32) | (k_pub >> 32));
    }
}

template <int NQ>
__device__ __forceinline__ void scan_mma(float (&acc)[NQ / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
    if constexpr (NQ == 16) wgmma_tf32_n16(acc, a, b, accumulate);
    else if constexpr (NQ == 32) wgmma_tf32_n32(acc, a, b, accumulate);
    else wgmma_tf32_n64(acc, a, b, accumulate);
}

// Accumulator element d[4 j + 2 h + e] of a thread is (row rsub + 8 h of its warpgroup's 64, query 8 j + 2 (lane % 4) + e).
template <int NQ>
__global__ void __launch_bounds__(kScanThreads, 1)
scan_rows_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_q, const ScanParams p) {
    constexpr int KD = kScanKD;
    constexpr int STAGE_BYTES = KD * kBoxBytes;
    constexpr int QBLK_BYTES = NQ * 128;                 // one K block of the query operand
    constexpr int NACC = NQ / 2;
    constexpr int ETH = 32 * kScanConsumerWarps;
    constexpr int EPW = kScanConsumerWarps;
    static_assert(NQ == 16 || NQ == 32 || NQ == 64, "queries per launch");

    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment by OFFSET (a pointer round-trip through an integer loses the shared address space)
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int KB = (p.dim + 31) / 32;                    // 128-byte K blocks
    const int NST = (KB + KD - 1) / KD;                  // pipeline stages per tile
    const int KBP = NST * KD;                            // K blocks the MMAs read: past KB (and past dim) TMA filled zeros
    uint8_t* qop = smem;
    uint8_t* ring = smem + KBP * QBLK_BYTES;
    uint8_t* state = ring + p.nstages * STAGE_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(state);
    uint64_t* empty = full + kScanMaxStages;
    uint64_t* qbar = empty + kScanMaxStages;
    float* tau_s = reinterpret_cast<float*>(state + 512);       // [NQ] running threshold of each query
    int* cnt_s = reinterpret_cast<int*>(state + 1024);          // [NQ] entries in each list of this CTA
    float* floor_s = reinterpret_cast<float*>(state + 1536);    // [NQ] largest score each list ever cut away

    int nq_live = p.nq;
    if (p.nq_dev != nullptr) {                           // second pass: nothing flagged in this launch's range -> nothing to do
        nq_live = min(p.nq, __ldg(p.nq_dev) - p.q_off);
        if (nq_live <= 0) return;                        // uniform over the grid: no barrier has been touched yet
    }
    const bool pool_mode = p.fixed_tau != nullptr;
    const int warp = threadIdx.x >> 5;
    const unsigned lane = lane_id();
    const int cta = blockIdx.x;

    if (threadIdx.x == 0) {
        for (int i = 0; i < p.nstages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], EPW); }
        mbar_init(qbar, 1);
        fence_mbar_init();
        prefetch_tmap(&tmap_x);
        prefetch_tmap(&tmap_q);
    }
    __syncthreads();

    if (warp == EPW) {
        // =========================== TMA producer ===========================
        if (elect_one()) {
            mbar_arrive_expect_tx(qbar, static_cast<uint32_t>(KBP * QBLK_BYTES));
            for (int kb = 0; kb < KBP; ++kb) tma_load_2d(qop + kb * QBLK_BYTES, &tmap_q, kb * 32, 0, qbar, kEvictLast);
            int slot = 0;
            uint32_t phase = 0;
            for (int t = cta; t < p.ntiles; t += gridDim.x) {
                for (int s = 0; s < NST; ++s) {
                    mbar_wait(&empty[slot], phase ^ 1);
                    mbar_arrive_expect_tx(&full[slot], STAGE_BYTES);
#pragma unroll
                    for (int kk = 0; kk < KD; ++kk) {
                        // K blocks past the row end are out of bounds: they arrive as zeros and still count their bytes
                        uint8_t* dst = ring + slot * STAGE_BYTES + kk * kBoxBytes;
                        tma_load_2d(dst, &tmap_x, (s * KD + kk) * 32, t * kTileRows, &full[slot], kEvictFirst);
                    }
                    if (++slot == p.nstages) { slot = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // =========================== consumers: MMA + epilogue ===========================
    const int wg = warp >> 2;                                // rows wg * 64 .. + 64 of every tile
    const int rsub = wg * 64 + (warp & 3) * 16 + static_cast<int>(lane >> 2);   // this thread's first row of the tile
    const int csub = 2 * static_cast<int>(lane & 3);
    const int et = threadIdx.x;                              // 0..ETH-1: per-query duties
    unsigned long long* mylists = p.lists + static_cast<size_t>(cta) * NQ * kListCap;
    const bool unit_rows = __uint_as_float(__ldg(p.stats_bits + 1)) < 1e-6f;
    const bool has_sc = p.metric == RMU_METRIC_COSINE && !unit_rows;
    const bool has_bi = p.metric == RMU_METRIC_L2 && !unit_rows;
    const bool qlive = et < NQ && et < nq_live;
    if (et < NQ) {
        tau_s[et] = qlive ? (pool_mode ? __ldg(p.fixed_tau + et) : -INFINITY) : INFINITY;
        cnt_s[et] = 0;
        floor_s[et] = -INFINITY;
    }
    bar_sync_named(1, ETH);
    mbar_wait(qbar, 0);                                      // the query operand is resident
    bool mine = false;                                       // this thread pushed a list past kListTrig
    int slot = 0;
    uint32_t phase = 0;
    int i = 0;
    for (int t = cta; t < p.ntiles; t += gridDim.x, ++i) {
        long long row[2];
        bool valid[2];
        float sc[2] = {1.f, 1.f}, bi[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {                        // issued before the MMAs: the loads hide behind them
            row[h] = static_cast<long long>(t) * kTileRows + rsub + 8 * h;
            valid[h] = row[h] < p.n;
            if (has_sc && valid[h]) sc[h] = __ldg(p.rscale + row[h]);
            if (has_bi && valid[h]) bi[h] = __ldg(p.rbias + row[h]);
        }
        float acc[NACC];
        int prev = -1;
        for (int s = 0; s < NST; ++s) {
            mbar_wait(&full[slot], phase);
            wgmma_fence();
            // no bounds test around the MMAs (a branch there makes ptxas serialise every wgmma): K steps past dim multiply
            // the zeros TMA wrote for out-of-bounds corpus columns and query columns, and add nothing
#pragma unroll
            for (int kk = 0; kk < KD; ++kk) {
                const uint64_t adesc = wgmma_desc_sw128(smem_u32(ring + slot * STAGE_BYTES + kk * kBoxBytes + wg * 64 * 128));
                const uint64_t bdesc = wgmma_desc_sw128(smem_u32(qop + (s * KD + kk) * QBLK_BYTES));
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t ko = static_cast<uint64_t>(k * 2);
                    scan_mma<NQ>(acc, adesc + ko, bdesc + ko, (s | kk | k) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                                 // the previous stage's MMAs have retired: its slot is free
            if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
            prev = slot;
            if (++slot == p.nstages) { slot = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);

        if (p.dbg != nullptr && i == 0 && cta < 2) {         // tiles 0 and 1 = the first 256 rows
#pragma unroll
            for (int j = 0; j < NACC; ++j) {
                const int ql = 8 * (j >> 2) + csub + (j & 1);
                if (ql < p.nq) p.dbg[ql * 2 * kTileRows + cta * kTileRows + rsub + 8 * ((j >> 1) & 1)] = acc[j];
            }
        }
        float v[NACC];
        unsigned m = 0u;
#pragma unroll
        for (int j = 0; j < NQ / 8; ++j) {
            const float2 tq = *reinterpret_cast<const float2*>(tau_s + 8 * j + csub);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int a = 4 * j + 2 * h;
                v[a] = fmaf(acc[a], sc[h], bi[h]);
                v[a + 1] = fmaf(acc[a + 1], sc[h], bi[h]);
                if (valid[h]) {
                    m |= (v[a] > tq.x) ? (1u << a) : 0u;
                    m |= (v[a + 1] > tq.y) ? (1u << (a + 1)) : 0u;
                }
            }
        }
        if (__any_sync(0xffffffffu, m != 0u)) {              // rare once the thresholds have risen
#pragma unroll
            for (int a = 0; a < NACC; ++a) {
                if (m & (1u << a)) {
                    const int ql = 8 * (a >> 2) + csub + (a & 1);
                    const uint32_t r = static_cast<uint32_t>(row[(a >> 1) & 1]);
                    if (pool_mode) {
                        const int pos = atomicAdd(p.pool_cnt + ql, 1);
                        if (pos < p.pool_cap) p.pool[static_cast<size_t>(ql) * p.pool_cap + pos] = make_key(v[a], r);
                    } else {
                        const int pos = atomicAdd(&cnt_s[ql], 1);
                        mylists[ql * kListCap + pos] = make_key(v[a], r);
                        mine |= pos >= kListTrig;
                    }
                }
            }
        }
        if (pool_mode) continue;
        // ---- tile boundary: sort + cut the lists that grew past kListTrig (every sort publishes the list's 16th key, so
        // the thresholds of all CTAs rise together: ~5 sorts per list over a 10M-row scan, most of them in the first tiles)
        const bool any = bar_red_or_named(1, ETH, mine);
        mine = false;
        if (any) {
            for (int ql = warp; ql < NQ; ql += EPW) {
                const int n = cnt_s[ql];
                if (n > kListTrig) {
                    unsigned long long* gslot = p.groups > 0 ? p.gmax + static_cast<size_t>(ql) * kGroupsMax + (cta % p.groups) : nullptr;
                    if (n <= 128) scan_sort_list<4>(mylists + ql * kListCap, n, cnt_s[ql], floor_s[ql], gslot, p.epoch);
                    else scan_sort_list<8>(mylists + ql * kListCap, n, cnt_s[ql], floor_s[ql], gslot, p.epoch);
                }
            }
            bar_sync_named(1, ETH);
        }
        // ---- refresh this query's threshold from what the other CTAs published
        if (qlive) {
            float tg = -INFINITY;
            if (p.groups > 0) {
                tg = INFINITY;
                const ulonglong2* g2 = reinterpret_cast<const ulonglong2*>(p.gmax + static_cast<size_t>(et) * kGroupsMax);
                for (int g = 0; g < p.groups; g += 2) {
                    const ulonglong2 w = __ldcg(g2 + (g >> 1));
                    const float s0 = static_cast<unsigned>(w.x >> 32) == p.epoch ? ordered_to_f32(static_cast<uint32_t>(w.x)) : -INFINITY;
                    const float s1 = static_cast<unsigned>(w.y >> 32) == p.epoch ? ordered_to_f32(static_cast<uint32_t>(w.y)) : -INFINITY;
                    tg = fminf(tg, fminf(s0, g + 1 < p.groups ? s1 : INFINITY));
                }
            }
            tau_s[et] = fmaxf(tg, floor_s[et]);
        }
    }
    if (et < NQ && !pool_mode) {                             // final: every tile ended with the barrier(s) above
        p.counts[cta * NQ + et] = cnt_s[et];
        p.floors[cta * NQ + et] = floor_s[et];
    }
}

// =====================================================================================================
// selection: union of the (cluster, query) lists -> best KSEL coarse candidates -> exact fp32 re-score ->
// sort -> top-k + certificate.  One CTA per query.
// =====================================================================================================
constexpr int kSel2Cap = 16384;                  // candidates gathered into shared memory (128 KB); more -> radix select over the lists

struct SelectParams {
    const unsigned long long* lists; const int* counts; const float* floors; const unsigned long long* gmax;
    int ncl, qb;               // lists per query (CTAs of the scan launch), list blocks per CTA (NQ)
    unsigned epoch; int groups;
    int ksel;                  // coarse candidates re-scored exactly (<= kSel2Max)
    const float* x; long long n; int dim; int metric;
    const float* q;            // [launch queries, dim]
    int q0;                    // index of the launch's first query in the outputs
    int k; long long id_offset;
    const unsigned* stats_bits;   // [0] max ||x|| , [1] max | ||x||^2 - 1 |
    float eps_rel;
    float* out_scores; long long* out_ids; int* flags;
    float* tau2;               // [nq] per query: the coarse-key threshold a second pass must use when the query is flagged
};

// exact_metric_multi with the four fmaf chains of one (query, row) pair spread over the four lanes of a quad (lane & 3 =
// chain): every chain sees the same elements in the same order and the partial sums are combined as (a0 + a1) + (a2 + a3),
// so the result is bit-identical to exact_metric_multi's.  All four lanes return the value.
__device__ __forceinline__ float exact_metric_quad(const float* __restrict__ q, const float* __restrict__ x, int D, int metric,
                                                   float qnorm) {
    const int c = static_cast<int>(lane_id() & 3u);
    const int D4 = D & ~3;
    float a = 0.f, nn = 0.f;
    if (metric == RMU_METRIC_L2) {
        for (int d = c; d < D4; d += 4) { const float e = q[d] - x[d]; a = fmaf(e, e, a); }
        if (c == 0) for (int d = D4; d < D; ++d) { const float e = q[d] - x[d]; a = fmaf(e, e, a); }
    } else {
        for (int d = c; d < D4; d += 4) {
            const float xv = x[d];
            a = fmaf(q[d], xv, a);
            if (metric == RMU_METRIC_COSINE) nn = fmaf(xv, xv, nn);
        }
        if (c == 0) for (int d = D4; d < D; ++d) {
            a = fmaf(q[d], x[d], a);
            if (metric == RMU_METRIC_COSINE) nn = fmaf(x[d], x[d], nn);
        }
    }
    const unsigned qb = lane_id() & ~3u;
    const float a0 = __shfl_sync(0xffffffffu, a, qb), a1 = __shfl_sync(0xffffffffu, a, qb + 1);
    const float a2 = __shfl_sync(0xffffffffu, a, qb + 2), a3 = __shfl_sync(0xffffffffu, a, qb + 3);
    const float s = (a0 + a1) + (a2 + a3);
    if (metric != RMU_METRIC_COSINE) return s;
    const float n0 = __shfl_sync(0xffffffffu, nn, qb), n1 = __shfl_sync(0xffffffffu, nn, qb + 1);
    const float n2 = __shfl_sync(0xffffffffu, nn, qb + 2), n3 = __shfl_sync(0xffffffffu, nn, qb + 3);
    const float xn = sqrtf((n0 + n1) + (n2 + n3));
    const float den = qnorm * xn;
    return den > 0.f ? s / den : 0.f;
}

// copy query q [dim] to shared memory and return ||q||, summed in the order of exact_scan_kernel (256 threads, stride 256,
// then block_sum) so that the cosine scores of the re-scores and of the exact scan are bit-identical.  All threads call.
__device__ __forceinline__ float stage_query(const float* __restrict__ q, int dim, float* qs, float* red /*[32]*/) {
    float part = 0.f;
    if (threadIdx.x < 256) {
        for (int d = threadIdx.x; d < dim; d += 256) {
            const float v = q[d];
            qs[d] = v;
            part = fmaf(v, v, part);
        }
    }
    return sqrtf(block_sum(part, red));
}

// exact re-score in place of keys[0 .. n): coarse key -> exact key of the same row, a quad of lanes per candidate (the
// same arithmetic as the exact scan: bit-identical scores).  All threads call.
__device__ __forceinline__ void rescore_keys(unsigned long long* keys, int n, const float* qs, float qnorm, const float* x, int dim,
                                             int metric) {
    const int tid = threadIdx.x;
    for (int c0 = 0; c0 < n; c0 += kSelThreads / 4) {
        const int c = c0 + (tid >> 2);
        const bool live = c < n;
        const uint32_t row = live ? key_row(keys[c]) : 0u;
        const float v = exact_metric_quad(qs, x + static_cast<long long>(row) * dim, dim, metric, qnorm);
        __syncwarp();
        if (live && (tid & 3) == 0) keys[c] = make_key(metric_to_rank(v, metric), row);
    }
}

__global__ void __launch_bounds__(kSelThreads) select_rescore_kernel(const SelectParams p) {
    __shared__ unsigned long long sel[kSel2Max];
    __shared__ int hist[256];
    __shared__ float red[32];
    __shared__ int s_n, s_nsel;
    __shared__ unsigned long long s_prefix;
    __shared__ int s_remaining, s_ties;
    __shared__ float s_tau;
    extern __shared__ unsigned long long sel_dyn[];  // cand [kSel2Cap], then the query [dim] floats
    unsigned long long* cand = sel_dyn;
    float* qs = reinterpret_cast<float*>(sel_dyn + kSel2Cap);

    const int f = blockIdx.x;
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;

    const float qnorm = stage_query(p.q + static_cast<long long>(f) * p.dim, p.dim, qs, red);

    // ---- what the scan may have rejected: everything <= tau (exchange) or <= a list's floor (cuts)
    if (tid == 0) {
        float tg = -INFINITY;
        if (p.groups > 0) {
            tg = INFINITY;
            for (int g = 0; g < p.groups; ++g) {
                const unsigned long long w = p.gmax[static_cast<size_t>(f) * kGroupsMax + g];
                tg = fminf(tg, static_cast<unsigned>(w >> 32) == p.epoch ? ordered_to_f32(static_cast<uint32_t>(w)) : -INFINITY);
            }
        }
        s_tau = tg;
        s_n = 0;
    }
    float fl = -INFINITY;
    for (int c = tid; c < p.ncl; c += blockDim.x) fl = fmaxf(fl, p.floors[c * p.qb + f]);
    for (int o = 16; o > 0; o >>= 1) fl = fmaxf(fl, __shfl_xor_sync(0xffffffffu, fl, o));
    __syncthreads();
    if (lane == 0) red[warp] = fl;
    __syncthreads();
    fl = red[0];
    for (int w = 1; w < kSelThreads / 32; ++w) fl = fmaxf(fl, red[w]);
    const float tau = s_tau;
    float bound = fmaxf(tau, fl);                // coarse upper bound of every row that is in no list
    __syncthreads();

    // ---- gather the entries above tau (two lists per warp step: the count loads of both are in flight together)
    for (int c = 2 * warp; c < p.ncl; c += 2 * (kSelThreads / 32)) {
        const int n0 = p.counts[c * p.qb + f];
        const int n1 = c + 1 < p.ncl ? p.counts[(c + 1) * p.qb + f] : 0;
        const unsigned long long* b0 = p.lists + static_cast<size_t>(c * p.qb + f) * kListCap;
        const unsigned long long* b1 = b0 + static_cast<size_t>(p.qb) * kListCap;
        for (int e = lane; e < n0 + n1; e += 32) {
            const unsigned long long key = e < n0 ? b0[e] : b1[e - n0];
            if (key_score(key) > tau) {
                const int pos = atomicAdd(&s_n, 1);
                if (pos < kSel2Cap) cand[pos] = key;
            }
        }
    }
    __syncthreads();
    const int n = s_n;
    int ncand;
    if (n <= p.ksel) {                           // every survivor is re-scored
        for (int i = tid; i < n; i += blockDim.x) sel[i] = cand[i];
        ncand = n;
    } else {
        // the ksel-th best key by radix select (shared memory when the survivors fit, else over the lists), then collect
        unsigned long long T;
        if (n <= kSel2Cap) {
            auto load_key = [&](long long idx) -> unsigned long long { return cand[idx]; };
            T = block_radix_select(load_key, n, p.ksel, hist, &s_prefix, &s_remaining, &s_ties);
            ncand = block_collect(load_key, n, T, sel, &s_nsel);
        } else {
            const long long total = static_cast<long long>(p.ncl) * kListCap;
            auto load_key = [&](long long idx) -> unsigned long long {
                const int c = static_cast<int>(idx / kListCap), e = static_cast<int>(idx % kListCap);
                if (e >= p.counts[c * p.qb + f]) return 0ull;
                const unsigned long long key = p.lists[static_cast<size_t>(c * p.qb + f) * kListCap + e];
                return key_score(key) > tau ? key : 0ull;
            };
            T = block_radix_select(load_key, total, p.ksel, hist, &s_prefix, &s_remaining, &s_ties);
            ncand = block_collect(load_key, total, T, sel, &s_nsel);
        }
        ncand = min(ncand, p.ksel);
        bound = fmaxf(bound, key_score(T));      // list entries that were not selected are below T
    }
    __syncthreads();

    rescore_keys(sel, ncand, qs, qnorm, p.x, p.dim, p.metric);
    block_sort_desc(sel, ncand);
    const int qg = p.q0 + f;
    write_topk(sel, ncand, qg, p.k, p.metric, p.id_offset, p.out_scores, p.out_ids);
    // ---- certificate: every row outside the candidate set has coarse key <= bound; its exact key is at
    //      most eps above.  The k-th exact candidate must beat that strictly.
    if (tid == 0 && p.flags != nullptr) {
        int flag = 0;
        if (bound > -INFINITY) {
            if (ncand < p.k) flag = 1;
            else {
                const float rk = key_score(sel[p.k - 1]);    // rank value of the k-th exact result
                const float xmax = __uint_as_float(p.stats_bits[0]);
                const bool unit = __uint_as_float(p.stats_bits[1]) < 1e-6f && p.metric != RMU_METRIC_IP;
                float kth_key, scale;                        // in the units of the coarse key
                if (p.metric == RMU_METRIC_IP) { kth_key = rk; scale = qnorm * xmax; }
                else if (p.metric == RMU_METRIC_COSINE) { kth_key = rk * qnorm; scale = qnorm; }
                else { kth_key = 0.5f * (qnorm * qnorm + rk) + (unit ? 0.5f : 0.f); scale = qnorm * xmax; }  // rk = -dist
                // unit rows: cosine / L2 keys were scanned as inner products, exact to 1e-6 (||x||^2 = 1 +- 1e-6)
                const float eps = p.eps_rel * scale + 1e-6f * (1.f + fabsf(kth_key)) + (unit ? 4e-6f * (1.f + qnorm) : 0.f);
                if (!(bound + eps < kth_key)) flag = 1;
                // every row whose exact score reaches the k-th candidate's has a coarse key above this:
                if (p.tau2 != nullptr) p.tau2[qg] = kth_key - eps - 1e-6f * (1.f + fabsf(kth_key));
            }
            if (flag && ncand < p.k && p.tau2 != nullptr) p.tau2[qg] = -INFINITY;   // not even k candidates: everything qualifies
        }
        p.flags[qg] = flag;
    }
}


// =====================================================================================================
// second pass for flagged queries: gather them, then (after the pool-mode scan) re-score their pools exactly
// =====================================================================================================
// block j < *nsel: copy flagged query qmap[j] into slot j of qbuf, its threshold into taubuf[j], clear its pool counter
__global__ void pool_prepare_kernel(const float* __restrict__ q, const int* __restrict__ qmap, const int* __restrict__ nsel, int dim,
                                    const float* __restrict__ tau2, float* __restrict__ qbuf, float* __restrict__ taubuf,
                                    int* __restrict__ pool_cnt) {
    const int j = blockIdx.x;
    if (j >= *nsel) return;
    const int qg = qmap[j];
    for (int d = threadIdx.x; d < dim; d += blockDim.x) qbuf[static_cast<size_t>(j) * dim + d] = q[static_cast<size_t>(qg) * dim + d];
    if (threadIdx.x == 0) { taubuf[j] = tau2[qg]; pool_cnt[j] = 0; }
}

struct PoolParams {
    unsigned long long* pool; const int* pool_cnt; int pool_cap;
    const int* qmap; const int* nsel;   // the grid has a block per slot: flagged queries beyond it stay flagged
    const float* x; int dim; int metric;
    const float* q;            // all queries [nq, dim]
    int k; long long id_offset;
    float* out_scores; long long* out_ids; int* flags;
};

// block j: every row of the pool (a superset of the rows whose exact score can reach the k-th) is re-scored exactly in
// place, the best k are selected; the result is the exact top-k.  A pool that overflowed leaves the query flagged.
__global__ void __launch_bounds__(kSelThreads) pool_rescore_kernel(const PoolParams p) {
    __shared__ unsigned long long sel[kSel2Max];
    __shared__ int hist[256];
    __shared__ float red[32];
    __shared__ int s_nsel;
    __shared__ unsigned long long s_prefix;
    __shared__ int s_remaining, s_ties;
    extern __shared__ float pqs[];               // [dim]
    const int j = blockIdx.x;
    if (j >= *p.nsel) return;
    const int qg = p.qmap[j];
    const int n = p.pool_cnt[j];
    if (n > p.pool_cap) return;                  // overflow: stays flagged, the exact scan answers
    const float qnorm = stage_query(p.q + static_cast<size_t>(qg) * p.dim, p.dim, pqs, red);
    unsigned long long* pool = p.pool + static_cast<size_t>(j) * p.pool_cap;
    rescore_keys(pool, n, pqs, qnorm, p.x, p.dim, p.metric);
    __syncthreads();
    auto load_key = [&](long long idx) -> unsigned long long { return pool[idx]; };
    const unsigned long long T = block_radix_select(load_key, n, p.k, hist, &s_prefix, &s_remaining, &s_ties);
    const int nsel = block_collect(load_key, n, T, sel, &s_nsel);
    block_sort_desc(sel, min(nsel, kSel2Max));   // everything collected is sorted, the best k are written
    write_topk(sel, min(nsel, p.k), qg, p.k, p.metric, p.id_offset, p.out_scores, p.out_ids);
    if (threadIdx.x == 0) p.flags[qg] = 0;       // answered exactly
}
