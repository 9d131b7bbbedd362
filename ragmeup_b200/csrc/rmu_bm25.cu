// Sparse leg of the hybrid retriever: Okapi BM25 scoring + top-n over an in-memory corpus (SURVEY.md §8 f2).
//
// The reference builds `BM25Retriever.from_texts(...)` (server/RAGHelper.py:436-443) — langchain-community's
// wrapper over rank_bm25.BM25Okapi — and queries it through the EnsembleRetriever (:501-503).  rank_bm25 scores a
// query in float64 numpy, one pass over ALL documents per query term:
//     score += idf[q] * (tf * (k1 + 1) / (tf + k1 * (1 - b + b * doc_len / avgdl)))
// and returns argsort(score)[::-1][:n].  Documents without the term add exactly 0, so the same float64 sums come out
// of an inverted index: here postings are CSR by term (documents ascending inside a term), `den[doc]` holds the
// document-length part `k1 * (1 - b + b * dl / avgdl)` computed by numpy on the host, and every float64 operation is
// issued with explicit round-to-nearest intrinsics in rank_bm25's order (no FMA contraction), terms in query order —
// scores are BIT-IDENTICAL to the numpy restatement in oracle/hybrid_ref.py.
//
// Kernel shape (HBM-latency-bound integer/fp64 gather work, no tensor cores): one CTA owns 4096 consecutive
// documents of one query, keeps their float64 scores in shared memory, walks the query's posting lists restricted to
// its document range (bounds found by one parallel binary search per term), then selects its k best in place
// (8-bit radix select on order-preserving keys, ties -> larger document index, which is what a stable argsort
// reversed yields).  A second kernel reduces the per-CTA candidates (4096 at a time) down to the final k, sorted.
#include <algorithm>
#include <mutex>
#include <vector>

#include "rmu_common.h"

namespace rmu {

constexpr int kBmDocs = 4096;       // documents (stage 1) or candidates (stage 2) per CTA
constexpr int kBmThreads = 256;
constexpr int kBmPer = kBmDocs / kBmThreads;   // consecutive items per thread in the order-preserving compaction
constexpr int kBmTermBatch = 256;   // query terms whose range bounds are resident at a time
constexpr int kBmMaxK = 256;
constexpr int kBmMaxQ = 65535;      // queries per launch: the query index is blockIdx.y

// order-preserving map double -> u64 (larger score = larger key); 0 is reserved for "absent"
__device__ __forceinline__ uint64_t f64_key(double v) {
    const uint64_t u = static_cast<uint64_t>(__double_as_longlong(v));
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_f64(uint64_t k) {
    const uint64_t u = (k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
    return __longlong_as_double(static_cast<long long>(u));
}

struct BmScratch {
    int hist[256];
    int warp_sums[kBmThreads / 32];
    unsigned long long prefix;     // radix-select: key prefix fixed so far
    int remaining;                 // radix-select: rank still to resolve inside the prefix bucket
    int total;                     // block_exclusive_scan: grand total
    int n_sel;
};

// exclusive prefix sum of one int per thread over the CTA (kBmThreads threads); total left in s->total
__device__ __forceinline__ int block_exclusive_scan(int v, BmScratch* s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();                      // previous users of warp_sums are done
    if (lane == 31) s->warp_sums[warp] = inc;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; ++w) base += s->warp_sums[w];
    if (threadIdx.x == kBmThreads - 1) s->total = base + inc;
    __syncthreads();
    return base + inc - v;
}

// Select the k best of the kBmDocs keys in shared memory (0 = absent).  Best = larger key; equal keys -> the LATER
// position wins.  Selected positions are written in ascending order to sel[0 .. n_sel).
__device__ void block_select(const uint64_t* key, int k, int* sel, BmScratch* s) {
    const int tid = threadIdx.x;
    // how many are present at all?
    int present = 0;
#pragma unroll
    for (int i = 0; i < kBmPer; ++i) present += key[tid * kBmPer + i] != 0;
    block_exclusive_scan(present, s);
    const int n_valid = s->total;
    uint64_t T = 1;     // threshold key: everything present is >= 1
    if (n_valid > k) {
        // k-th largest key by 8 passes of 8 bits, most significant first
        if (tid == 0) { s->prefix = 0; s->remaining = k; }
        __syncthreads();
        for (int pass = 0; pass < 8; ++pass) {
            const int shift = 56 - 8 * pass;
            for (int i = tid; i < 256; i += kBmThreads) s->hist[i] = 0;
            __syncthreads();
            const unsigned long long pre = s->prefix;
            const unsigned long long mask = pass == 0 ? 0ull : (~0ull << (shift + 8));
            for (int i = tid; i < kBmDocs; i += kBmThreads) {
                const uint64_t kk = key[i];
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
                s->remaining = rem;                 // rank inside bucket b
                s->prefix = pre | (static_cast<unsigned long long>(b) << shift);
            }
            __syncthreads();
        }
        T = s->prefix;
    }
    // r ties (key == T) are taken, counted from the END of the position order
    int gt = 0, tie = 0;
#pragma unroll
    for (int i = 0; i < kBmPer; ++i) {
        const uint64_t kk = key[tid * kBmPer + i];
        gt += kk > T;
        tie += kk == T && kk != 0;
    }
    block_exclusive_scan(gt, s);
    const int n_gt = s->total;
    int tie_before = block_exclusive_scan(tie, s);
    const int n_tie = s->total;
    const int r = n_valid > k ? k - n_gt : n_tie;      // n_valid <= k: T = 1 -> take every tie as well
    const int first_tie = n_tie - r;                   // tie ranks >= first_tie are selected
    int mine = 0;
    unsigned flags = 0;
#pragma unroll
    for (int i = 0; i < kBmPer; ++i) {
        const uint64_t kk = key[tid * kBmPer + i];
        bool take = kk > T;
        if (kk == T && kk != 0) { take = tie_before >= first_tie; ++tie_before; }
        if (take) { flags |= 1u << i; ++mine; }
    }
    int off = block_exclusive_scan(mine, s);
    if (tid == kBmThreads - 1) s->n_sel = s->total;
#pragma unroll
    for (int i = 0; i < kBmPer; ++i)
        if (flags & (1u << i)) sel[off++] = tid * kBmPer + i;
    __syncthreads();
}

__device__ __forceinline__ long long lower_bound_doc(const int32_t* __restrict__ post_doc, long long lo, long long hi, long long doc) {
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (static_cast<long long>(post_doc[mid]) < doc) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// stage 1: scores of documents [blockIdx.x * 4096, +4096) for query blockIdx.y, then the CTA's k best
__global__ void __launch_bounds__(kBmThreads)
bm25_score_kernel(const long long* __restrict__ post_ptr, const int32_t* __restrict__ post_doc,
                  const int32_t* __restrict__ post_tf, const double* __restrict__ den, const double* __restrict__ idf,
                  double k1p1, long long n_docs, const int32_t* __restrict__ q_ptr, const int32_t* __restrict__ q_terms,
                  int k, double* __restrict__ cand_score, int32_t* __restrict__ cand_idx) {
    __shared__ unsigned long long cell[kBmDocs];      // float64 score bits while scoring, then the order-preserving key
    __shared__ long long t_lo[kBmTermBatch];
    __shared__ int t_len[kBmTermBatch];
    __shared__ double t_idf[kBmTermBatch];
    __shared__ int sel[kBmMaxK];
    __shared__ BmScratch scratch;
    const int tid = threadIdx.x;
    const long long d0 = static_cast<long long>(blockIdx.x) * kBmDocs;
    const int nd = static_cast<int>(min(static_cast<long long>(kBmDocs), n_docs - d0));
    for (int i = tid; i < kBmDocs; i += kBmThreads) cell[i] = 0ull;      // bits of +0.0
    const int qs = q_ptr[blockIdx.y], qe = q_ptr[blockIdx.y + 1];
    for (int tb = qs; tb < qe; tb += kBmTermBatch) {
        const int bs = min(kBmTermBatch, qe - tb);
        __syncthreads();
        if (tid < bs) {
            const int term = q_terms[tb + tid];
            const long long p0 = post_ptr[term], p1 = post_ptr[term + 1];
            const long long lo = lower_bound_doc(post_doc, p0, p1, d0);
            // one posting per (term, document): at most nd postings fall in this CTA's range
            const long long hi = lower_bound_doc(post_doc, lo, min(p1, lo + nd), d0 + nd);
            t_lo[tid] = lo;
            t_len[tid] = static_cast<int>(hi - lo);
            t_idf[tid] = idf[term];
        }
        __syncthreads();
        for (int j = 0; j < bs; ++j) {
            const int len = t_len[j];
            if (len == 0) continue;                   // uniform: read from shared memory
            const long long lo = t_lo[j];
            const double w = t_idf[j];
            for (int p = tid; p < len; p += kBmThreads) {
                const int doc = post_doc[lo + p];
                const double tf = static_cast<double>(post_tf[lo + p]);
                // idf * (tf * (k1 + 1) / (tf + k1 * (1 - b + b * dl / avgdl))), rank_bm25's operation order
                const double val = __dmul_rn(w, __ddiv_rn(__dmul_rn(tf, k1p1), __dadd_rn(tf, den[doc])));
                const int slot = doc - static_cast<int>(d0);
                // one posting per (term, document): no two threads touch the same slot within a term
                cell[slot] = static_cast<unsigned long long>(__double_as_longlong(__dadd_rn(__longlong_as_double(static_cast<long long>(cell[slot])), val)));
            }
            __syncthreads();                          // next term may touch the same documents
        }
    }
    __syncthreads();
    uint64_t* key = reinterpret_cast<uint64_t*>(cell);
    for (int i = tid; i < kBmDocs; i += kBmThreads)
        key[i] = i < nd ? f64_key(__longlong_as_double(static_cast<long long>(cell[i]))) : 0ull;
    __syncthreads();
    block_select(key, k, sel, &scratch);
    const int n_sel = scratch.n_sel;
    const size_t out = (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * k;
    for (int i = tid; i < k; i += kBmThreads) {
        if (i < n_sel) {
            cand_score[out + i] = key_f64(key[sel[i]]);
            cand_idx[out + i] = static_cast<int32_t>(d0 + sel[i]);
        } else {
            cand_score[out + i] = 0.0;
            cand_idx[out + i] = -1;
        }
    }
}

// stage 2: k best of candidates [blockIdx.x * 4096, +4096) of query blockIdx.y (candidate lists are in ascending
// document order).  The last round (one CTA per query) writes them sorted: score descending, ties -> larger index.
__global__ void __launch_bounds__(kBmThreads)
bm25_select_kernel(const double* __restrict__ in_score, const int32_t* __restrict__ in_idx, int m, int k, int final_round,
                   double* __restrict__ out_score, int32_t* __restrict__ out_idx, double* __restrict__ res_score,
                   long long* __restrict__ res_ids) {
    __shared__ uint64_t key[kBmDocs];
    __shared__ int sel[kBmMaxK];
    __shared__ int32_t sel_idx[kBmMaxK];
    __shared__ BmScratch scratch;
    const int tid = threadIdx.x;
    const int c0 = blockIdx.x * kBmDocs;
    const size_t base = static_cast<size_t>(blockIdx.y) * m + c0;
    for (int i = tid; i < kBmDocs; i += kBmThreads) {
        uint64_t kk = 0;
        if (c0 + i < m && in_idx[base + i] >= 0) kk = f64_key(in_score[base + i]);
        key[i] = kk;
    }
    __syncthreads();
    block_select(key, k, sel, &scratch);
    const int n_sel = scratch.n_sel;
    if (!final_round) {
        const size_t out = (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * k;
        for (int i = tid; i < k; i += kBmThreads) {
            out_score[out + i] = i < n_sel ? key_f64(key[sel[i]]) : 0.0;
            out_idx[out + i] = i < n_sel ? in_idx[base + sel[i]] : -1;
        }
        return;
    }
    for (int i = tid; i < n_sel; i += kBmThreads) sel_idx[i] = in_idx[base + sel[i]];
    __syncthreads();
    const size_t out = static_cast<size_t>(blockIdx.y) * k;
    for (int i = tid; i < k; i += kBmThreads) {
        if (i < n_sel) {
            const uint64_t ki = key[sel[i]];
            const int32_t di = sel_idx[i];
            int rank = 0;
            for (int j = 0; j < n_sel; ++j) {
                const uint64_t kj = key[sel[j]];
                rank += kj > ki || (kj == ki && sel_idx[j] > di);
            }
            res_score[out + rank] = key_f64(ki);
            res_ids[out + rank] = di;
        } else {
            res_score[out + i] = 0.0;
            res_ids[out + i] = -1;
        }
    }
}

}  // namespace rmu

using namespace rmu;

struct rmu_bm25 {
    int64_t n_docs = 0, n_terms = 0, nnz = 0;
    double k1p1 = 2.5;
    int device = 0;
    long long* post_ptr = nullptr;
    int32_t *post_doc = nullptr, *post_tf = nullptr;
    double *den = nullptr, *idf = nullptr;
    // workspace (grown on demand): candidate ping-pong buffers + host-call staging
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
    Buf cs[2], ci[2], qptr, qterms, out_s, out_i;
    std::mutex mu;
};

template <typename T>
static int bm_upload(T** dst, const T* src_h, size_t n) {
    RMU_CUDA(cudaMalloc(reinterpret_cast<void**>(dst), std::max<size_t>(n, 1) * sizeof(T)));
    if (n) RMU_CUDA(cudaMemcpy(*dst, src_h, n * sizeof(T), cudaMemcpyHostToDevice));
    return RMU_OK;
}

// Select rounds over candidate lists in[Q, m] (ascending document order, index -1 = absent) down to the sorted top k in
// out_scores / out_ids [Q, k].  Round r writes ws_s[r & 1] / ws_i[r & 1], each of Q * ceil(m / 4096) * k elements; every
// round but the last hands its output to the next as input.  Q <= kBmMaxQ.
static int bm25_select_rounds(const double* in_s, const int32_t* in_i, int Q, int m, int k, double* const ws_s[2],
                              int32_t* const ws_i[2], double* out_scores, int64_t* out_ids, cudaStream_t st) {
    for (int r = 0;; ++r) {
        const int blocks = (m + kBmDocs - 1) / kBmDocs;
        const int final_round = blocks == 1;
        bm25_select_kernel<<<dim3(static_cast<unsigned>(blocks), static_cast<unsigned>(Q)), kBmThreads, 0, st>>>(
            in_s, in_i, m, k, final_round, ws_s[r & 1], ws_i[r & 1], out_scores, reinterpret_cast<long long*>(out_ids));
        count_launch();
        RMU_CHECK_LAUNCH();
        if (final_round) return RMU_OK;
        in_s = ws_s[r & 1];
        in_i = ws_i[r & 1];
        m = blocks * k;
    }
}

static int bm25_search_locked(rmu_bm25* h, const int32_t* q_ptr, const int32_t* q_terms, int Q, int k, double* out_scores,
                              int64_t* out_ids, cudaStream_t st) {
    const int nblk = static_cast<int>((h->n_docs + kBmDocs - 1) / kBmDocs);
    // the query index is gridDim.y (at most 65 535): larger batches run in chunks, each reusing the candidate buffers
    const size_t need = static_cast<size_t>(std::min(Q, kBmMaxQ)) * nblk * k;
    for (int i = 0; i < 2; ++i) {
        int rc = h->cs[i].ensure(need * sizeof(double));
        if (rc == RMU_OK) rc = h->ci[i].ensure(need * sizeof(int32_t));
        if (rc != RMU_OK) return rc;
    }
    // stage 1 writes buffer 0; the rounds then go 0 -> 1 -> 0 -> ...
    double* const ws_s[2] = {h->cs[1].as<double>(), h->cs[0].as<double>()};
    int32_t* const ws_i[2] = {h->ci[1].as<int32_t>(), h->ci[0].as<int32_t>()};
    ProfScope _ps(PROF_MISC, st);
    for (int q0 = 0; q0 < Q; q0 += kBmMaxQ) {
        const int qc = std::min(kBmMaxQ, Q - q0);
        bm25_score_kernel<<<dim3(static_cast<unsigned>(nblk), static_cast<unsigned>(qc)), kBmThreads, 0, st>>>(
            h->post_ptr, h->post_doc, h->post_tf, h->den, h->idf, h->k1p1, h->n_docs, q_ptr + q0, q_terms, k,
            h->cs[0].as<double>(), h->ci[0].as<int32_t>());
        count_launch();
        RMU_CHECK_LAUNCH();
        const size_t o = static_cast<size_t>(q0) * k;
        const int rc = bm25_select_rounds(h->cs[0].as<double>(), h->ci[0].as<int32_t>(), qc, nblk * k, k, ws_s, ws_i,
                                          out_scores + o, out_ids + o, st);
        if (rc != RMU_OK) return rc;
    }
    return RMU_OK;
}

extern "C" {

int rmu_bm25_create(int64_t n_docs, int64_t n_terms, const int64_t* post_ptr_h, const int32_t* post_doc_h,
                    const int32_t* post_tf_h, const double* den_h, const double* idf_h, double k1_plus_1, rmu_bm25** out) {
    if (!out || n_docs <= 0 || n_terms < 0 || !post_ptr_h || !den_h || (n_terms > 0 && (!idf_h || !post_doc_h || !post_tf_h))) {
        set_error("rmu_bm25_create: bad argument");
        return RMU_ERR_ARG;
    }
    if (n_docs > 0x7FFFFFFFll - kBmDocs) { set_error("rmu_bm25_create: more than 2^31 documents"); return RMU_ERR_UNSUPPORTED; }
    const int64_t nnz = post_ptr_h[n_terms];
    for (int64_t t = 0; t < n_terms; ++t) {
        if (post_ptr_h[t + 1] < post_ptr_h[t]) { set_error("rmu_bm25_create: post_ptr must be non-decreasing"); return RMU_ERR_ARG; }
    }
    rmu_bm25* h = new rmu_bm25();
    h->n_docs = n_docs; h->n_terms = n_terms; h->nnz = nnz; h->k1p1 = k1_plus_1;
    if (cudaGetDevice(&h->device) != cudaSuccess) {
        set_error("rmu_bm25_create: no CUDA device (this library has no CPU path)");
        delete h;
        return RMU_ERR_CUDA;
    }
    static_assert(sizeof(long long) == sizeof(int64_t), "int64");
    int rc = bm_upload(&h->post_ptr, reinterpret_cast<const long long*>(post_ptr_h), static_cast<size_t>(n_terms) + 1);
    if (rc == RMU_OK) rc = bm_upload(&h->post_doc, post_doc_h, static_cast<size_t>(nnz));
    if (rc == RMU_OK) rc = bm_upload(&h->post_tf, post_tf_h, static_cast<size_t>(nnz));
    if (rc == RMU_OK) rc = bm_upload(&h->den, den_h, static_cast<size_t>(n_docs));
    if (rc == RMU_OK) rc = bm_upload(&h->idf, idf_h, static_cast<size_t>(n_terms));
    if (rc != RMU_OK) { rmu_bm25_destroy(h); return rc; }
    *out = h;
    return RMU_OK;
}

int rmu_bm25_destroy(rmu_bm25* h) {
    if (!h) return RMU_OK;
    cudaFree(h->post_ptr); cudaFree(h->post_doc); cudaFree(h->post_tf); cudaFree(h->den); cudaFree(h->idf);
    for (int i = 0; i < 2; ++i) { cudaFree(h->cs[i].p); cudaFree(h->ci[i].p); }
    cudaFree(h->qptr.p); cudaFree(h->qterms.p); cudaFree(h->out_s.p); cudaFree(h->out_i.p);
    delete h;
    return RMU_OK;
}

int64_t rmu_bm25_size(const rmu_bm25* h) { return h ? h->n_docs : 0; }
int64_t rmu_bm25_terms(const rmu_bm25* h) { return h ? h->n_terms : 0; }

static int bm25_check(const rmu_bm25* h, const void* q_ptr, const void* out_s, const void* out_i, int Q, int k) {
    if (!h || !q_ptr || !out_s || !out_i || Q <= 0) { set_error("rmu_bm25_search: bad argument"); return RMU_ERR_ARG; }
    if (k < 1 || k > kBmMaxK) { set_error("rmu_bm25_search: k must be in [1, 256]"); return RMU_ERR_UNSUPPORTED; }
    return RMU_OK;
}

int rmu_bm25_search(rmu_bm25* h, const int32_t* q_ptr, const int32_t* q_terms, int Q, int k, double* out_scores,
                    int64_t* out_ids, void* stream) {
    int rc = bm25_check(h, q_ptr, out_scores, out_ids, Q, k);
    if (rc != RMU_OK) return rc;
    std::lock_guard<std::mutex> g(h->mu);
    return bm25_search_locked(h, q_ptr, q_terms, Q, k, out_scores, out_ids, static_cast<cudaStream_t>(stream));
}

int rmu_bm25_search_host(rmu_bm25* h, const int32_t* q_ptr_h, const int32_t* q_terms_h, int Q, int k, double* out_scores_h,
                         int64_t* out_ids_h, void* stream) {
    int rc = bm25_check(h, q_ptr_h, out_scores_h, out_ids_h, Q, k);
    if (rc != RMU_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::lock_guard<std::mutex> g(h->mu);
    const int nt = q_ptr_h[Q];
    if (nt < 0 || q_ptr_h[0] != 0) { set_error("rmu_bm25_search_host: q_ptr must start at 0 and be non-decreasing"); return RMU_ERR_ARG; }
    for (int i = 0; i < nt; ++i) {
        if (q_terms_h[i] < 0 || q_terms_h[i] >= h->n_terms) { set_error("rmu_bm25_search_host: term id out of range"); return RMU_ERR_ARG; }
    }
    rc = h->qptr.ensure((static_cast<size_t>(Q) + 1) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->qterms.ensure(static_cast<size_t>(nt) * sizeof(int32_t));
    if (rc == RMU_OK) rc = h->out_s.ensure(static_cast<size_t>(Q) * k * sizeof(double));
    if (rc == RMU_OK) rc = h->out_i.ensure(static_cast<size_t>(Q) * k * sizeof(int64_t));
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(h->qptr.p, q_ptr_h, (static_cast<size_t>(Q) + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (nt) RMU_CUDA(cudaMemcpyAsync(h->qterms.p, q_terms_h, static_cast<size_t>(nt) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    rc = bm25_search_locked(h, h->qptr.as<int32_t>(), h->qterms.as<int32_t>(), Q, k, h->out_s.as<double>(), h->out_i.as<int64_t>(), st);
    if (rc != RMU_OK) return rc;
    RMU_CUDA(cudaMemcpyAsync(out_scores_h, h->out_s.p, static_cast<size_t>(Q) * k * sizeof(double), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaMemcpyAsync(out_ids_h, h->out_i.p, static_cast<size_t>(Q) * k * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    RMU_CUDA(cudaStreamSynchronize(st));
    return RMU_OK;
}

/* For tests: the select rounds alone on caller-owned candidate lists (see the header) */
int rmu_debug_bm25_select(const double* scores, const int32_t* idx, int Q, int m, int k, double* ws_scores,
                          int32_t* ws_idx, int64_t ws_elems, double* out_scores, int64_t* out_ids, void* stream) {
    if (!scores || !idx || !ws_scores || !ws_idx || !out_scores || !out_ids || Q < 1 || m < 1) {
        set_error("rmu_debug_bm25_select: bad argument");
        return RMU_ERR_ARG;
    }
    if (k < 1 || k > kBmMaxK || Q > kBmMaxQ) {
        set_error("rmu_debug_bm25_select: k must be in [1, 256] and Q at most 65535");
        return RMU_ERR_UNSUPPORTED;
    }
    const int64_t half = static_cast<int64_t>(Q) * ((m + kBmDocs - 1) / kBmDocs) * k;
    if (ws_elems < 2 * half) {
        set_error("rmu_debug_bm25_select: workspace needs 2 * Q * ceil(m / 4096) * k elements");
        return RMU_ERR_ARG;
    }
    double* const ws_s[2] = {ws_scores, ws_scores + half};
    int32_t* const ws_i[2] = {ws_idx, ws_idx + half};
    return bm25_select_rounds(scores, idx, Q, m, k, ws_s, ws_i, out_scores, out_ids, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
