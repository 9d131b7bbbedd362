// Sparse leg of the Postgres configuration: pg_search BM25 scoring, boolean clauses, phrases and top-k over an
// appendable inverted index with positions.
//
// The reference's PostgresBM25Retriever (server/PostgresBM25Retriever.py, built at server/RAGHelper.py:445-462) runs
// `content @@@ '<query>' ORDER BY paradedb.score DESC LIMIT k` against ParadeDB's pg_search, which scores with
// tantivy's Bm25Weight in float32:
//     clause score = weight * (tf / (tf + cache[fieldnorm_id]))
// weight = (sum of the clause's term idfs) * (1 + K1) and the 256-entry `cache` (document-length part per fieldnorm
// id) are computed by numpy on the host (ragmeup_b200/pg_search.py); this file only adds, multiplies and divides,
// each with an explicit round-to-nearest intrinsic (no FMA contraction), and sums a document's matched MUST / SHOULD
// clauses in clause order, so scores are BIT-IDENTICAL to the float32 restatement in oracle/pg_bm25_ref.py.
//
// Index: immutable segments, each a CSR by term over a contiguous range of global rows (rows ascending inside a
// term; per posting tf and the start of its sorted position list) plus a fieldnorm byte per row.  A global alive
// bitmap masks deleted rows.  The host appends segments and merges the trailing ones geometrically (pg_bm25.py).
//
// Kernel shape (latency-bound gather work, no tensor cores), as rmu_bm25.cu: one CTA owns 4096 consecutive rows of
// one segment for one query, keeps their float32 scores, MUST counts and flags in shared memory and walks each
// clause's postings restricted to its rows (bounds by one binary search per clause term).  A phrase walks the
// postings of its rarest term (the host orders a phrase's terms by document frequency) and counts the positions at
// which every other term sits at its offset.  Then the CTA selects its k best by an 8-bit radix select on 64-bit keys
// (score key << 32 | ~row), which are unique, so ties go to the lower row without a tie rule; a second kernel reduces
// the candidates down to the final k, sorted.
#include <algorithm>
#include <mutex>
#include <vector>

#include "rmu_common.h"

namespace rmu {

constexpr int kPgRows = 4096;       // rows (stage 1) or candidates (stage 2) per CTA
constexpr int kPgThreads = 256;
constexpr int kPgPer = kPgRows / kPgThreads;
constexpr int kPgMaxK = 256;
constexpr int kPgMaxQ = 65535;      // queries per launch: the query index is blockIdx.y
constexpr int kPgMaxPhrase = 128;   // tokens in one clause
constexpr int kPgMaxMust = 65535;   // MUST clauses in one query: the count lives in 16 bits of the row state

constexpr uint32_t kStShould = 1u << 16;
constexpr uint32_t kStNot = 1u << 17;

enum { kShould = 0, kMust = 1, kMustNot = 2 };

struct PgSeg {
    const long long* post_ptr;      // [n_terms + 1]
    const int32_t* post_row;        // [nnz] row within the segment, ascending inside a term
    const int32_t* post_tf;         // [nnz]
    const long long* pos_start;     // [nnz] first position of the posting in `pos`
    const int32_t* pos;             // [sum tf] ascending inside a posting
    const uint8_t* fnorm;           // [n_rows] fieldnorm id
    long long n_terms;              // term ids >= n_terms have no postings here
    int row0;                       // global row of local row 0
    int n_rows;
};

struct PgScratch {
    int hist[256];
    int warp_sums[kPgThreads / 32];
    unsigned long long prefix;
    int remaining;
    int total;
    int n_sel;
    int n_must;
};

__device__ __forceinline__ int pg_exclusive_scan(int v, PgScratch* s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) s->warp_sums[warp] = inc;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; ++w) base += s->warp_sums[w];
    if (threadIdx.x == kPgThreads - 1) s->total = base + inc;
    __syncthreads();
    return base + inc - v;
}

// The min(k, present) largest of kPgRows unique keys (0 = absent); positions in ascending order to sel[0 .. n_sel).
__device__ __forceinline__ void pg_block_select(const unsigned long long* key, int k, int* sel, PgScratch* s) {
    const int tid = threadIdx.x;
    int present = 0;
#pragma unroll
    for (int i = 0; i < kPgPer; ++i) present += key[tid * kPgPer + i] != 0;
    pg_exclusive_scan(present, s);
    unsigned long long T = 1;
    if (s->total > k) {
        if (tid == 0) { s->prefix = 0; s->remaining = k; }
        __syncthreads();
        for (int pass = 0; pass < 8; ++pass) {
            const int shift = 56 - 8 * pass;
            for (int i = tid; i < 256; i += kPgThreads) s->hist[i] = 0;
            __syncthreads();
            const unsigned long long pre = s->prefix;
            const unsigned long long mask = pass == 0 ? 0ull : (~0ull << (shift + 8));
            for (int i = tid; i < kPgRows; i += kPgThreads) {
                const unsigned long long kk = key[i];
                if (kk != 0 && (kk & mask) == pre) atomicAdd(&s->hist[(kk >> shift) & 0xFF], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int rem = s->remaining;
                int b = 255;
                for (; b > 0; --b) {
                    if (s->hist[b] >= rem) break;
                    rem -= s->hist[b];
                }
                s->remaining = rem;
                s->prefix = pre | (static_cast<unsigned long long>(b) << shift);
            }
            __syncthreads();
        }
        T = s->prefix;              // the k-th largest key itself: keys are unique
    }
    int mine = 0;
    unsigned flags = 0;
#pragma unroll
    for (int i = 0; i < kPgPer; ++i) {
        if (key[tid * kPgPer + i] >= T) { flags |= 1u << i; ++mine; }
    }
    int off = pg_exclusive_scan(mine, s);
    if (tid == kPgThreads - 1) s->n_sel = s->total;
#pragma unroll
    for (int i = 0; i < kPgPer; ++i)
        if (flags & (1u << i)) sel[off++] = tid * kPgPer + i;
    __syncthreads();
}

__device__ __forceinline__ long long pg_lower_bound(const int32_t* __restrict__ a, long long lo, long long hi, int v) {
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ bool pg_contains(const int32_t* __restrict__ a, long long lo, long long hi, int v) {
    lo = pg_lower_bound(a, lo, hi, v);
    return lo < hi && a[lo] == v;
}

__device__ __forceinline__ unsigned long long pg_key(float score, int row) {
    const uint32_t u = __float_as_uint(score);
    const uint32_t f = (u >> 31) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(f) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<uint32_t>(row));
}
__device__ __forceinline__ float pg_key_score(unsigned long long k) {
    const uint32_t f = static_cast<uint32_t>(k >> 32);
    return __uint_as_float((f >> 31) ? (f & 0x7FFFFFFFu) : ~f);
}
__device__ __forceinline__ long long pg_key_row(unsigned long long k) {
    return static_cast<long long>(0xFFFFFFFFu - static_cast<uint32_t>(k & 0xFFFFFFFFull));
}

// stage 1: rows [blk.y, +4096) of segment blk.x for query blockIdx.y, then the CTA's k best keys
// at most 85 registers: three CTAs per SM (shared memory allows five); the default bound spills
__global__ void __launch_bounds__(kPgThreads, 3)
pgbm25_score_kernel(const PgSeg* __restrict__ segs, const int2* __restrict__ blk, const uint32_t* __restrict__ alive,
                    const float* __restrict__ cache, const int32_t* __restrict__ q_ptr, const int32_t* __restrict__ c_occur,
                    const float* __restrict__ c_weight, const int32_t* __restrict__ c_tptr,
                    const int32_t* __restrict__ ct_term, const int32_t* __restrict__ ct_off, int k,
                    unsigned long long* __restrict__ cand) {
    // a row's score and state share the 8 bytes its key replaces, so each thread converts its own rows in place
    __shared__ union {
        struct { float score; uint32_t state; } cell[kPgRows];
        unsigned long long key[kPgRows];
    } u;
    __shared__ long long t_lo[kPgMaxPhrase];
    __shared__ int t_len[kPgMaxPhrase];
    __shared__ int t_off[kPgMaxPhrase];
    __shared__ float s_cache[256];
    __shared__ int sel[kPgMaxK];
    __shared__ PgScratch scratch;
    __shared__ int s_skip;
    const int tid = threadIdx.x;
    const int2 b = blk[blockIdx.x];
    const PgSeg* sg = segs + b.x;
    const int r0 = b.y;
    const int nr = min(kPgRows, sg->n_rows - r0);
    const long long n_terms = sg->n_terms;
    const long long* __restrict__ post_ptr = sg->post_ptr;
    const int32_t* __restrict__ post_row = sg->post_row;
    const int32_t* __restrict__ post_tf = sg->post_tf;
    const long long* __restrict__ pos_start = sg->pos_start;
    const int32_t* __restrict__ pos = sg->pos;
    const uint8_t* __restrict__ fnorm = sg->fnorm;
    for (int i = tid; i < kPgRows; i += kPgThreads) { u.cell[i].score = 0.0f; u.cell[i].state = 0u; }
    s_cache[tid] = cache[tid];
    const int qs = q_ptr[blockIdx.y], qe = q_ptr[blockIdx.y + 1];
    if (tid == 0) {
        int m = 0;
        for (int c = qs; c < qe; ++c) m += c_occur[c] == kMust;
        scratch.n_must = m;
    }
    for (int c = qs; c < qe; ++c) {
        const int t0 = c_tptr[c], nt = c_tptr[c + 1] - t0;
        __syncthreads();                              // the previous clause is done with t_* and the row state
        if (tid == 0) s_skip = 0;
        __syncthreads();
        if (tid < nt) {
            const int term = ct_term[t0 + tid];
            long long lo = 0, len = 0;
            if (term < n_terms) {
                const long long p0 = post_ptr[term], p1 = post_ptr[term + 1];
                lo = pg_lower_bound(post_row, p0, p1, r0);
                // one posting per (term, row): at most nr postings fall in this CTA's rows
                len = pg_lower_bound(post_row, lo, min(p1, lo + nr), r0 + nr) - lo;
            }
            t_lo[tid] = lo;
            t_len[tid] = static_cast<int>(len);
            t_off[tid] = ct_off[t0 + tid];
            if (len == 0) s_skip = 1;                 // a phrase missing a term matches no row here
        }
        __syncthreads();
        if (s_skip) continue;                         // uniform: read from shared memory
        const int occur = c_occur[c];
        const float w = c_weight[c];
        const long long lo0 = t_lo[0];
        const int len0 = t_len[0], off0 = t_off[0];
        for (int p = tid; p < len0; p += kPgThreads) {
            const long long e = lo0 + p;
            const int row = post_row[e];
            int tf = post_tf[e];
            if (nt > 1) {
                bool all = true;
                for (int j = 1; j < nt && all; ++j) all = pg_contains(post_row, t_lo[j], t_lo[j] + t_len[j], row);
                int count = 0;
                if (all) {
                    const long long x0 = pos_start[e];
                    for (int i = 0; i < tf; ++i) {
                        const int base = pos[x0 + i] - off0;
                        bool hit = true;
                        for (int j = 1; j < nt && hit; ++j) {
                            const long long ej = pg_lower_bound(post_row, t_lo[j], t_lo[j] + t_len[j], row);
                            const long long xj = pos_start[ej];
                            hit = pg_contains(pos, xj, xj + post_tf[ej], base + t_off[j]);
                        }
                        count += hit;
                    }
                }
                tf = count;
            }
            if (tf == 0) continue;
            const int slot = row - r0;
            // one posting per (term, row): no two threads touch the same slot within a clause
            if (occur == kMustNot) {
                u.cell[slot].state |= kStNot;
            } else {
                const float tff = static_cast<float>(tf);
                const float sc = __fmul_rn(w, __fdiv_rn(tff, __fadd_rn(tff, s_cache[fnorm[row]])));
                u.cell[slot].score = __fadd_rn(u.cell[slot].score, sc);
                u.cell[slot].state += occur == kMust ? 1u : 0u;
                if (occur == kShould) u.cell[slot].state |= kStShould;
            }
        }
    }
    __syncthreads();
    const uint32_t n_must = static_cast<uint32_t>(scratch.n_must);
    const int grow0 = sg->row0 + r0;
    for (int slot = tid; slot < kPgRows; slot += kPgThreads) {
        unsigned long long kk = 0ull;
        if (slot < nr) {
            const uint32_t st = u.cell[slot].state;
            const int g = grow0 + slot;
            const bool live = (alive[g >> 5] >> (g & 31)) & 1u;
            const bool match = (st & 0xFFFFu) == n_must && (n_must > 0 || (st & kStShould)) && !(st & kStNot);
            if (live && match) kk = pg_key(u.cell[slot].score, g);
        }
        u.key[slot] = kk;
    }
    __syncthreads();
    pg_block_select(u.key, k, sel, &scratch);
    const int n_sel = scratch.n_sel;
    const size_t out = (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * k;
    for (int i = tid; i < k; i += kPgThreads) cand[out + i] = i < n_sel ? u.key[sel[i]] : 0ull;
}

// stage 2: k best of candidate keys [blockIdx.x * 4096, +4096) of query blockIdx.y; the last round (one CTA per
// query) writes them sorted, score descending (ties: lower row, already inside the key)
__global__ void __launch_bounds__(kPgThreads)
pgbm25_select_kernel(const unsigned long long* __restrict__ in, int m, int k, int final_round,
                     unsigned long long* __restrict__ out, float* __restrict__ res_score, long long* __restrict__ res_row) {
    __shared__ unsigned long long key[kPgRows];
    __shared__ int sel[kPgMaxK];
    __shared__ PgScratch scratch;
    const int tid = threadIdx.x;
    const int c0 = blockIdx.x * kPgRows;
    const size_t base = static_cast<size_t>(blockIdx.y) * m + c0;
    for (int i = tid; i < kPgRows; i += kPgThreads) key[i] = c0 + i < m ? in[base + i] : 0ull;
    __syncthreads();
    pg_block_select(key, k, sel, &scratch);
    const int n_sel = scratch.n_sel;
    if (!final_round) {
        const size_t o = (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * k;
        for (int i = tid; i < k; i += kPgThreads) out[o + i] = i < n_sel ? key[sel[i]] : 0ull;
        return;
    }
    const size_t o = static_cast<size_t>(blockIdx.y) * k;
    for (int i = tid; i < k; i += kPgThreads) {
        if (i < n_sel) {
            const unsigned long long ki = key[sel[i]];
            int rank = 0;
            for (int j = 0; j < n_sel; ++j) rank += key[sel[j]] > ki;
            res_score[o + rank] = pg_key_score(ki);
            res_row[o + rank] = pg_key_row(ki);
        } else {
            res_score[o + i] = 0.0f;
            res_row[o + i] = -1;
        }
    }
}

}  // namespace rmu

using namespace rmu;

struct rmu_pgbm25 {
    struct Seg {
        PgSeg d{};                  // device pointers
        void* bufs[6] = {};
        int64_t nnz = 0;
    };
    struct Buf {
        void* p = nullptr;
        size_t bytes = 0;
        int ensure(size_t need) {
            if (p && need <= bytes) return RMU_OK;
            if (p) { RMU_CUDA(cudaFree(p)); p = nullptr; bytes = 0; }
            RMU_CUDA(cudaMalloc(&p, std::max<size_t>(need, 16)));
            bytes = std::max<size_t>(need, 16);
            return RMU_OK;
        }
        template <typename T> T* as() const { return static_cast<T*>(p); }
    };
    int device = 0;
    std::vector<Seg> segs;
    int64_t rows_end = 0;           // one past the last global row of any segment
    int64_t alive_words = 0;        // words of the bitmap uploaded by the last set_alive
    bool layout_dirty = true;       // segment table / block table need a re-upload
    int nblk = 0;
    Buf alive, seg_tab, blk_tab, cand[2], qptr, cocc, cw, ctp, ctt, cto, cache, out_s, out_r;
    std::mutex mu;
};

static void pg_free_seg(rmu_pgbm25::Seg& s) {
    for (void*& p : s.bufs) { cudaFree(p); p = nullptr; }
}

template <typename T>
static int pg_upload(void** dst, const T* src_h, size_t n) {
    RMU_CUDA(cudaMalloc(dst, std::max<size_t>(n, 1) * sizeof(T)));
    if (n) RMU_CUDA(cudaMemcpy(*dst, src_h, n * sizeof(T), cudaMemcpyHostToDevice));
    return RMU_OK;
}

static int pg_layout(rmu_pgbm25* h) {
    if (!h->layout_dirty) return RMU_OK;
    std::vector<PgSeg> tab;
    std::vector<int2> blk;
    for (size_t s = 0; s < h->segs.size(); ++s) {
        tab.push_back(h->segs[s].d);
        for (int r = 0; r < h->segs[s].d.n_rows; r += kPgRows) blk.push_back(make_int2(static_cast<int>(s), r));
    }
    h->nblk = static_cast<int>(blk.size());
    int rc = h->seg_tab.ensure(std::max<size_t>(tab.size(), 1) * sizeof(PgSeg));
    if (rc == RMU_OK) rc = h->blk_tab.ensure(std::max<size_t>(blk.size(), 1) * sizeof(int2));
    if (rc != RMU_OK) return rc;
    if (!tab.empty()) RMU_CUDA(cudaMemcpy(h->seg_tab.p, tab.data(), tab.size() * sizeof(PgSeg), cudaMemcpyHostToDevice));
    if (!blk.empty()) RMU_CUDA(cudaMemcpy(h->blk_tab.p, blk.data(), blk.size() * sizeof(int2), cudaMemcpyHostToDevice));
    h->layout_dirty = false;
    return RMU_OK;
}

extern "C" {

int rmu_pgbm25_create(rmu_pgbm25** out) {
    if (!out) { set_error("rmu_pgbm25_create: bad argument"); return RMU_ERR_ARG; }
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        set_error("rmu_pgbm25_create: no CUDA device (this library has no CPU path)");
        return RMU_ERR_CUDA;
    }
    rmu_pgbm25* h = new rmu_pgbm25();
    h->device = dev;
    *out = h;
    return RMU_OK;
}

int rmu_pgbm25_destroy(rmu_pgbm25* h) {
    if (!h) return RMU_OK;
    for (auto& s : h->segs) pg_free_seg(s);
    rmu_pgbm25::Buf* bufs[] = {&h->alive, &h->seg_tab, &h->blk_tab, &h->cand[0], &h->cand[1], &h->qptr, &h->cocc,
                               &h->cw, &h->ctp, &h->ctt, &h->cto, &h->cache, &h->out_s, &h->out_r};
    for (auto* b : bufs) cudaFree(b->p);
    delete h;
    return RMU_OK;
}

int rmu_pgbm25_push_segment(rmu_pgbm25* h, int64_t row0, int64_t n_rows, int64_t n_terms, const int64_t* post_ptr_h,
                            const int32_t* post_row_h, const int32_t* post_tf_h, const int64_t* pos_start_h,
                            const int32_t* pos_h, const uint8_t* fnorm_h) {
    if (!h || row0 < 0 || n_rows < 1 || n_terms < 0 || !post_ptr_h || !fnorm_h) {
        set_error("rmu_pgbm25_push_segment: bad argument");
        return RMU_ERR_ARG;
    }
    if (row0 + n_rows > 0x7FFFFFFFll - kPgRows) { set_error("rmu_pgbm25_push_segment: more than 2^31 rows"); return RMU_ERR_UNSUPPORTED; }
    std::lock_guard<std::mutex> g(h->mu);
    if (row0 < h->rows_end) { set_error("rmu_pgbm25_push_segment: rows must follow the last segment's"); return RMU_ERR_ARG; }
    const int64_t nnz = post_ptr_h[n_terms];
    if (post_ptr_h[0] != 0 || nnz < 0 || (nnz > 0 && (!post_row_h || !post_tf_h || !pos_start_h || !pos_h))) {
        set_error("rmu_pgbm25_push_segment: bad postings");
        return RMU_ERR_ARG;
    }
    int64_t n_pos = 0;
    for (int64_t t = 0; t < n_terms; ++t) {
        if (post_ptr_h[t + 1] < post_ptr_h[t]) { set_error("rmu_pgbm25_push_segment: post_ptr must be non-decreasing"); return RMU_ERR_ARG; }
    }
    for (int64_t e = 0; e < nnz; ++e) {
        if (post_row_h[e] < 0 || post_row_h[e] >= n_rows || post_tf_h[e] < 1 || pos_start_h[e] != n_pos) {
            set_error("rmu_pgbm25_push_segment: posting out of range");
            return RMU_ERR_ARG;
        }
        n_pos += post_tf_h[e];
    }
    rmu_pgbm25::Seg s;
    int rc = pg_upload(&s.bufs[0], reinterpret_cast<const long long*>(post_ptr_h), static_cast<size_t>(n_terms) + 1);
    if (rc == RMU_OK) rc = pg_upload(&s.bufs[1], post_row_h, static_cast<size_t>(nnz));
    if (rc == RMU_OK) rc = pg_upload(&s.bufs[2], post_tf_h, static_cast<size_t>(nnz));
    if (rc == RMU_OK) rc = pg_upload(&s.bufs[3], reinterpret_cast<const long long*>(pos_start_h), static_cast<size_t>(nnz));
    if (rc == RMU_OK) rc = pg_upload(&s.bufs[4], pos_h, static_cast<size_t>(n_pos));
    if (rc == RMU_OK) rc = pg_upload(&s.bufs[5], fnorm_h, static_cast<size_t>(n_rows));
    if (rc != RMU_OK) { pg_free_seg(s); return rc; }
    s.d = PgSeg{static_cast<const long long*>(s.bufs[0]), static_cast<const int32_t*>(s.bufs[1]),
                static_cast<const int32_t*>(s.bufs[2]), static_cast<const long long*>(s.bufs[3]),
                static_cast<const int32_t*>(s.bufs[4]), static_cast<const uint8_t*>(s.bufs[5]), n_terms,
                static_cast<int>(row0), static_cast<int>(n_rows)};
    s.nnz = nnz;
    h->segs.push_back(s);
    h->rows_end = row0 + n_rows;
    h->layout_dirty = true;
    return RMU_OK;
}

int rmu_pgbm25_pop_segments(rmu_pgbm25* h, int n) {
    if (!h || n < 0) { set_error("rmu_pgbm25_pop_segments: bad argument"); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> g(h->mu);
    if (static_cast<size_t>(n) > h->segs.size()) { set_error("rmu_pgbm25_pop_segments: fewer segments than that"); return RMU_ERR_ARG; }
    RMU_CUDA(cudaDeviceSynchronize());            // a search on another stream may still read them
    for (int i = 0; i < n; ++i) { pg_free_seg(h->segs.back()); h->segs.pop_back(); }
    h->rows_end = h->segs.empty() ? 0 : static_cast<int64_t>(h->segs.back().d.row0) + h->segs.back().d.n_rows;
    h->layout_dirty = true;
    return RMU_OK;
}

int rmu_pgbm25_segments(const rmu_pgbm25* h) { return h ? static_cast<int>(h->segs.size()) : 0; }

int rmu_pgbm25_set_alive(rmu_pgbm25* h, const uint32_t* words_h, int64_t n_words) {
    if (!h || n_words < 0 || (n_words > 0 && !words_h)) { set_error("rmu_pgbm25_set_alive: bad argument"); return RMU_ERR_ARG; }
    std::lock_guard<std::mutex> g(h->mu);
    const size_t bytes = static_cast<size_t>(n_words) * sizeof(uint32_t);
    if (h->alive.p && bytes > h->alive.bytes) RMU_CUDA(cudaDeviceSynchronize());
    int rc = h->alive.ensure(bytes);
    if (rc != RMU_OK) return rc;
    if (bytes) RMU_CUDA(cudaMemcpy(h->alive.p, words_h, bytes, cudaMemcpyHostToDevice));
    h->alive_words = n_words;
    return RMU_OK;
}

int rmu_pgbm25_search_host(rmu_pgbm25* h, int Q, const int32_t* q_ptr_h, const int32_t* c_occur_h, const float* c_weight_h,
                           const int32_t* c_tptr_h, const int32_t* ct_term_h, const int32_t* ct_off_h, const float* cache_h,
                           int k, float* out_scores_h, int64_t* out_rows_h, void* stream) {
    if (!h || Q < 1 || !q_ptr_h || !cache_h || !out_scores_h || !out_rows_h) { set_error("rmu_pgbm25_search_host: bad argument"); return RMU_ERR_ARG; }
    if (k < 1 || k > kPgMaxK) { set_error("rmu_pgbm25_search_host: k must be in [1, 256]"); return RMU_ERR_UNSUPPORTED; }
    const int nc = q_ptr_h[Q];
    if (q_ptr_h[0] != 0 || nc < 0 || (nc > 0 && (!c_occur_h || !c_weight_h || !c_tptr_h || !ct_term_h || !ct_off_h))) {
        set_error("rmu_pgbm25_search_host: q_ptr must start at 0");
        return RMU_ERR_ARG;
    }
    for (int q = 0; q < Q; ++q) {
        if (q_ptr_h[q + 1] < q_ptr_h[q]) { set_error("rmu_pgbm25_search_host: q_ptr must be non-decreasing"); return RMU_ERR_ARG; }
        int must = 0;
        for (int c = q_ptr_h[q]; c < q_ptr_h[q + 1]; ++c) must += c_occur_h[c] == kMust;
        if (must > kPgMaxMust) { set_error("rmu_pgbm25_search_host: more than 65535 MUST clauses in a query"); return RMU_ERR_UNSUPPORTED; }
    }
    const int nt = nc > 0 ? c_tptr_h[nc] : 0;
    for (int c = 0; c < nc; ++c) {
        const int len = c_tptr_h[c + 1] - c_tptr_h[c];
        if (c_occur_h[c] < kShould || c_occur_h[c] > kMustNot || len < 1 || len > kPgMaxPhrase || c_tptr_h[0] != 0) {
            set_error("rmu_pgbm25_search_host: a clause needs an occur in 0..2 and 1..128 terms");
            return RMU_ERR_ARG;
        }
    }
    for (int i = 0; i < nt; ++i) {
        if (ct_term_h[i] < 0) { set_error("rmu_pgbm25_search_host: negative term id"); return RMU_ERR_ARG; }
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::lock_guard<std::mutex> g(h->mu);
    if (h->alive_words * 32 < h->rows_end) { set_error("rmu_pgbm25_search_host: the alive bitmap does not cover every row"); return RMU_ERR_ARG; }
    int rc = pg_layout(h);
    if (rc != RMU_OK) return rc;
    const size_t qk = static_cast<size_t>(Q) * k;
    if (h->nblk == 0) {                            // no rows: no matches
        std::fill(out_scores_h, out_scores_h + qk, 0.0f);
        std::fill(out_rows_h, out_rows_h + qk, int64_t(-1));
        return RMU_OK;
    }
    const size_t need = static_cast<size_t>(std::min(Q, kPgMaxQ)) * h->nblk * k * sizeof(unsigned long long);
    rc = h->cand[0].ensure(need);
    if (rc == RMU_OK) rc = h->cand[1].ensure(need);
    if (rc == RMU_OK) rc = h->qptr.ensure((static_cast<size_t>(Q) + 1) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->cocc.ensure(static_cast<size_t>(nc) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->cw.ensure(static_cast<size_t>(nc) * sizeof(float));
    if (rc == RMU_OK) rc = h->ctp.ensure((static_cast<size_t>(nc) + 1) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->ctt.ensure(static_cast<size_t>(nt) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->cto.ensure(static_cast<size_t>(nt) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->cache.ensure(256 * sizeof(float));
    if (rc == RMU_OK) rc = h->out_s.ensure(qk * sizeof(float));
    if (rc == RMU_OK) rc = h->out_r.ensure(qk * sizeof(int64_t));
    if (rc != RMU_OK) return rc;
    const int32_t zero = 0;
    RMU_CUDA(cudaMemcpyAsync(h->qptr.p, q_ptr_h, (static_cast<size_t>(Q) + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (nc) {
        RMU_CUDA(cudaMemcpyAsync(h->cocc.p, c_occur_h, static_cast<size_t>(nc) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        RMU_CUDA(cudaMemcpyAsync(h->cw.p, c_weight_h, static_cast<size_t>(nc) * sizeof(float), cudaMemcpyHostToDevice, st));
        RMU_CUDA(cudaMemcpyAsync(h->ctp.p, c_tptr_h, (static_cast<size_t>(nc) + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        RMU_CUDA(cudaMemcpyAsync(h->ctt.p, ct_term_h, static_cast<size_t>(nt) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        RMU_CUDA(cudaMemcpyAsync(h->cto.p, ct_off_h, static_cast<size_t>(nt) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    } else {
        RMU_CUDA(cudaMemcpyAsync(h->ctp.p, &zero, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    }
    RMU_CUDA(cudaMemcpyAsync(h->cache.p, cache_h, 256 * sizeof(float), cudaMemcpyHostToDevice, st));
    ProfScope _ps(PROF_MISC, st);
    for (int q0 = 0; q0 < Q; q0 += kPgMaxQ) {
        const int qc = std::min(kPgMaxQ, Q - q0);
        pgbm25_score_kernel<<<dim3(static_cast<unsigned>(h->nblk), static_cast<unsigned>(qc)), kPgThreads, 0, st>>>(
            h->seg_tab.as<PgSeg>(), h->blk_tab.as<int2>(), h->alive.as<uint32_t>(), h->cache.as<float>(),
            h->qptr.as<int32_t>() + q0, h->cocc.as<int32_t>(), h->cw.as<float>(), h->ctp.as<int32_t>(),
            h->ctt.as<int32_t>(), h->cto.as<int32_t>(), k, h->cand[0].as<unsigned long long>());
        count_launch();
        RMU_CHECK_LAUNCH();
        const unsigned long long* in = h->cand[0].as<unsigned long long>();
        int m = h->nblk * k;
        for (int r = 0;; ++r) {
            const int blocks = (m + kPgRows - 1) / kPgRows;
            const int final_round = blocks == 1;
            unsigned long long* o = h->cand[(r + 1) & 1].as<unsigned long long>();
            pgbm25_select_kernel<<<dim3(static_cast<unsigned>(blocks), static_cast<unsigned>(qc)), kPgThreads, 0, st>>>(
                in, m, k, final_round, o, h->out_s.as<float>() + static_cast<size_t>(q0) * k,
                h->out_r.as<long long>() + static_cast<size_t>(q0) * k);
            count_launch();
            RMU_CHECK_LAUNCH();
            if (final_round) break;
            in = o;
            m = blocks * k;
        }
    }
    RMU_CUDA(cudaMemcpyAsync(out_scores_h, h->out_s.p, qk * sizeof(float), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaMemcpyAsync(out_rows_h, h->out_r.p, qk * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    return RMU_OK;
}

}  // extern "C"
