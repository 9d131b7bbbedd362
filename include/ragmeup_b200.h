/*
 * ragmeup_b200 — C ABI of the H100-native dense-retrieval hot path.
 *
 * The reference (AI-Commandos/RAGMeUp) is pure Python and reaches this path through
 * three LangChain objects owned by RAGHelper (SURVEY.md §8b):
 *   self.embeddings  HuggingFaceEmbeddings      server/RAGHelper_local.py:114-117, RAGHelper_cloud.py:101-103
 *   self.db          Milvus / PGVector          server/RAGHelper.py:388-394, 399-404, 431, 497-499, 525
 *   self.compressor  ScoredCrossEncoderReranker(HuggingFaceCrossEncoder)
 *                                               server/RAGHelper.py:483-486, server/ScoredCrossEncoderReranker.py:25-45
 * There is no FFI in the reference; the binding a maintainer adds is the ctypes stub in
 * INTEGRATION.md (ragmeup_b200/_lib.py is that stub).  Each entry point below names the
 * reference interface it stands behind.
 *
 * Conventions: plain C, opaque handles, int return codes (0 = ok, <0 = error, text from
 * rmu_last_error()), every pointer is a DEVICE pointer unless its name ends in _h, every
 * asynchronous call takes the cudaStream_t to run on (as void*), no hidden device syncs unless
 * stated.  Handles own the corpus / weights and their scratch memory; callers own inputs and
 * outputs.  All calls on one handle are serialised internally (Flask worker threads share one
 * RAGHelper: server/server.py:141-146,394).
 */
#ifndef RAGMEUP_B200_H
#define RAGMEUP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RMU_OK 0
#define RMU_ERR_ARG -1
#define RMU_ERR_CUDA -2
#define RMU_ERR_UNSUPPORTED -3
#define RMU_ERR_RANGE -4         /* an activation left the range its storage can hold (Qwen3's fp16 planes) */
#define RMU_ERR_BUSY -5          /* a decode session has no free row, or its KV cache cannot grow while rows are live */

/* metric ids — Milvus FLAT/L2 is the reference default store metric (langchain-milvus 0.1.3
 * via server/RAGHelper.py:388-394); PGVector uses cosine distance (server/RAGHelper.py:399-404). */
#define RMU_METRIC_IP 0      /* score = <q,x>            larger is better  */
#define RMU_METRIC_COSINE 1  /* score = cos(q,x)         larger is better  */
#define RMU_METRIC_L2 2      /* score = ||q-x||^2        smaller is better */

/* search modes */
#define RMU_SEARCH_AUTO 0    /* wgmma coarse scan + exact fp32 re-score + certified fallback */
#define RMU_SEARCH_EXACT 1   /* fp32 CUDA-core scan only (what AUTO falls back to)            */
#define RMU_SEARCH_TENSOR_NOFALLBACK 2 /* diagnostics: coarse+re-score, flags reported, no fallback */

const char* rmu_last_error(void);
int rmu_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t rmu_launch_count(void);

/* per-kernel-class device timing (CUDA events on the launching stream; used by bench.py for the
 * roofline objects).  classes: 0 scan, 1 finalize, 2 exact scan, 3 merge, 4 gemm, 5 attention,
 * 6 layernorm, 7 embedding, 8 pool/head, 9 misc, 10 second-pass scan launches (queries whose certificate failed; exit at once when there are none),
 * 11 decode attention and KV cache writes, 12 LM head (its GEMM is also in 4), 13 sampler, 14 the NF4 kernels
 * (quantiser, dequantiser, decode GEMV; the prefill's E1 GEMMs on dequantised weights stay in 4).  rmu_profile_read synchronises the recorded events. */
void rmu_profile_enable(int on);
void rmu_profile_reset(void);
int rmu_profile_read(int cls, double* total_ms, int64_t* launches);

/* ------------------------------------------------------------------ flat vector index
 * Stands behind the vector store: Milvus.from_documents / PGVector ctor (RAGHelper.py:385-404),
 * db.add_documents (:431,525) and the retriever's col.search (:497-499). */
typedef struct rmu_index rmu_index;

int rmu_index_create(int dim, int metric, rmu_index** out);
void rmu_index_destroy(rmu_index* idx);
int rmu_index_reserve(rmu_index* idx, int64_t rows);
/* append n rows of `dim` fp32; src_is_host selects a host (pinned or pageable) source */
int rmu_index_add(rmu_index* idx, const float* vecs, int64_t n, int src_is_host, void* stream);
/* overwrite existing rows in place (PGVector's upsert-on-id, langchain-postgres add_embeddings): rows[n] int64 local row
 * numbers and vecs [n, dim] fp32, both DEVICE pointers; rows outside [0, size) are ignored */
int rmu_index_set_rows(rmu_index* idx, const int64_t* rows, const float* vecs, int64_t n, void* stream);
/* delete rows (a vector store's delete by id / by expression): rows_h[n] int64 local row numbers, a HOST array, in any
 * order, duplicates allowed (taken as a set).  The surviving rows close up in place on the device, keeping their order,
 * and their statistics are recomputed: afterwards the index equals a fresh one built by adding the survivors in order.
 * Capacity is kept.  A null rows_h with n > 0, n < 0 or a row outside [0, size) returns RMU_ERR_ARG before any CUDA
 * call, with the index untouched; n = 0 launches nothing.  Waits for all work on the device (like a growing add), so
 * nothing enqueued earlier reads rows while they move. */
int rmu_index_remove(rmu_index* idx, const int64_t* rows_h, int64_t n, void* stream);
int64_t rmu_index_size(const rmu_index* idx);
int rmu_index_dim(const rmu_index* idx);
int rmu_index_metric(const rmu_index* idx);
int rmu_index_clear(rmu_index* idx);
/* raw device pointer to the [size, dim] fp32 corpus (persistence / tests) */
const float* rmu_index_data(const rmu_index* idx);

/* top-k of every query against the whole index.
 *   queries [nq, dim] fp32, out_scores [nq, k] fp32, out_ids [nq, k] int64 = id_offset + row,
 *   missing results (k > size) are id -1 with score -inf (+inf for L2).
 *   stats_h (nullable, host int32[4]): {queries whose certificate failed in the first tensor pass, first-pass
 *   tensor-scan launches, queries that still needed the exact fp32 CUDA-core scan after the second pass, 0};
 *   requesting it makes the call synchronise the stream. */
int rmu_index_search(rmu_index* idx, const float* queries, int nq, int k, int64_t id_offset, int mode,
                     float* out_scores, int64_t* out_ids, int32_t* stats_h, void* stream);
/* same, HOST buffers in and out (H2D + D2H inside the call, synchronises `stream`) */
int rmu_index_search_host(rmu_index* idx, const float* queries_h, int nq, int k, int64_t id_offset, int mode,
                          float* out_scores_h, int64_t* out_ids_h, void* stream);
/* For tests: raw TF32 accumulators of the scan's first 256 rows (tiles 0 and 1, one per CTA) -> out [nq, 256] device
 * fp32 (rows past size() are written as 0).  dim % 4 == 0 and nq <= the scan's query block at this dim (64 up to
 * dim 384, 32 up to 768, 16 up to 1536); queries [nq, dim] device fp32, 16-byte aligned.  Shapes outside that, an
 * empty index or a null pointer return RMU_ERR_ARG before any CUDA call. */
int rmu_debug_scan_tile(rmu_index* idx, const float* queries, int nq, float* out, void* stream);
/* rows[n] (int64, local row numbers) -> out [n, dim]; feeds MMR (langchain-milvus fetches the
 * fetch_k stored vectors the same way after col.search) */
int rmu_index_gather(rmu_index* idx, const int64_t* rows, int n, float* out, void* stream);

/* merge R per-shard result lists (after the NCCL all-gather): [R, nq, k] -> [nq, k] */
int rmu_topk_merge(const float* scores, const int64_t* ids, int R, int nq, int k, int metric,
                   float* out_scores, int64_t* out_ids, void* stream);

/* the same on the buffer ONE all-gather fills: rank r's scores start at scores + r * rank_stride_scores (elements),
 * its ids at ids + r * rank_stride_ids, so a per-rank record {scores[nq*k], ids[nq*k]} needs no repacking */
int rmu_topk_merge_strided(const float* scores, const int64_t* ids, int64_t rank_stride_scores, int64_t rank_stride_ids,
                           int R, int nq, int k, int metric, float* out_scores, int64_t* out_ids, void* stream);

/* greedy maximal-marginal-relevance re-selection (langchain `maximal_marginal_relevance`,
 * used by as_retriever(search_type="mmr"), server/RAGHelper.py:497-499,533-535):
 * q [nq, dim], cand [nq, fetch_k, dim], n_cand[nq] valid candidates, out_sel [nq, k] int32
 * positions into the candidate list (-1 padded).  lambda_mult is a double, as the Python float langchain multiplies
 * with: rounding 0.3 to float moves it by 1.2e-8, which is enough to flip a near-tie. */
int rmu_mmr_select(const float* q, const float* cand, const int32_t* n_cand, int nq, int fetch_k, int dim,
                   int k, double lambda_mult, int32_t* out_sel, void* stream);

/* cosine DISTANCE (1 - cosine similarity) between consecutive rows of x [n, dim] -> out [n - 1] (device, float64):
 * the sentence-to-sentence distances of langchain_experimental's SemanticChunker, which the reference builds at
 * server/RAGHelper.py:329-341 and runs through text_splitter.split_documents (:368) (SURVEY.md §8 f4).  A zero row has
 * similarity 0 (cosine_similarity maps NaN and +-inf to 0), so its distances are exactly 1. */
int rmu_adjacent_cosine_distance(const float* x, int64_t n, int dim, double* out, void* stream);

/* ------------------------------------------------------------------ BM25 sparse leg (SURVEY.md §8 f2)
 * Stands behind langchain_community.retrievers.BM25Retriever (rank_bm25.BM25Okapi.get_scores /
 * get_top_n), built at server/RAGHelper.py:436-443 and queried through the EnsembleRetriever
 * (:501-503).  The inverted index is CSR by term: postings of term t are
 * post_doc/post_tf[post_ptr[t] .. post_ptr[t+1]) with documents ascending; den[d] =
 * k1 * (1 - b + b * doc_len[d] / avgdl) and idf[t] are float64, computed by the host exactly as
 * rank_bm25 does.  Scores are float64 and bit-identical to rank_bm25's; results are ordered score
 * descending, equal scores by larger document index (numpy stable argsort reversed). */
typedef struct rmu_bm25 rmu_bm25;
int rmu_bm25_create(int64_t n_docs, int64_t n_terms, const int64_t* post_ptr_h, const int32_t* post_doc_h,
                    const int32_t* post_tf_h, const double* den_h, const double* idf_h, double k1_plus_1,
                    rmu_bm25** out);                    /* host arrays, copied to the device */
int rmu_bm25_destroy(rmu_bm25* h);
int64_t rmu_bm25_size(const rmu_bm25* h);
int64_t rmu_bm25_terms(const rmu_bm25* h);
/* Q queries: terms of query i are q_terms[q_ptr[i] .. q_ptr[i+1]) (term ids in query order, repeats
 * kept); out_scores [Q, k] float64, out_ids [Q, k] int64 document numbers, -1 padded when the corpus
 * has fewer than k documents.  1 <= k <= 256; any Q >= 1 (batches past 65 535 queries run in chunks).  Device pointers: */
int rmu_bm25_search(rmu_bm25* h, const int32_t* q_ptr, const int32_t* q_terms, int Q, int k, double* out_scores,
                    int64_t* out_ids, void* stream);
/* the same with HOST buffers (copies + synchronise inside the call) */
int rmu_bm25_search_host(rmu_bm25* h, const int32_t* q_ptr_h, const int32_t* q_terms_h, int Q, int k,
                         double* out_scores_h, int64_t* out_ids_h, void* stream);

/* Host-only helper (no GPU work): the inverted index rank_bm25 would build from
 * `[text.split() for text in texts]` (BM25Retriever.from_texts, server/RAGHelper.py:436-443) — Python
 * str.split() whitespace semantics on UTF-8, vocabulary ids in first-seen order, postings CSR by term
 * with documents ascending.  texts_utf8[i] has text_bytes[i] bytes (no terminator needed). */
typedef struct rmu_bm25_csr rmu_bm25_csr;
int rmu_bm25_csr_build(const char* const* texts_utf8, const int64_t* text_bytes, int64_t n_docs, rmu_bm25_csr** out);
int rmu_bm25_csr_sizes(const rmu_bm25_csr* c, int64_t* n_terms, int64_t* nnz, int64_t* vocab_bytes);
/* doc_len [n_docs], post_ptr [n_terms+1], post_doc/post_tf [nnz], vocab_off [n_terms+1], vocab_bytes */
int rmu_bm25_csr_export(const rmu_bm25_csr* c, int64_t* doc_len, int64_t* post_ptr, int32_t* post_doc,
                        int32_t* post_tf, int64_t* vocab_off, char* vocab_bytes);
int rmu_bm25_csr_free(rmu_bm25_csr* c);

/* ------------------------------------------------------------------ pg_search BM25 (Postgres sparse leg)
 * Stands behind the reference's PostgresBM25Retriever (server/PostgresBM25Retriever.py, server/RAGHelper.py:445-462):
 * `content @@@ '<query>' ORDER BY paradedb.score DESC LIMIT k`, tantivy's float32 Bm25Weight.  The index is a list of
 * immutable segments over consecutive global rows: postings CSR by term (rows within the segment ascending inside a
 * term, tf >= 1 and a position list per posting, pos_start[e] = sum of the earlier tfs), a fieldnorm id per row, and
 * one alive bitmap over all global rows (bit r of word r / 32).  The host appends segments and drops trailing ones to
 * replace them by their merge. */
typedef struct rmu_pgbm25 rmu_pgbm25;
int rmu_pgbm25_create(rmu_pgbm25** out);
int rmu_pgbm25_destroy(rmu_pgbm25* h);
/* rows [row0, row0 + n_rows) after every row of the existing segments; host arrays, copied to the device */
int rmu_pgbm25_push_segment(rmu_pgbm25* h, int64_t row0, int64_t n_rows, int64_t n_terms, const int64_t* post_ptr_h,
                            const int32_t* post_row_h, const int32_t* post_tf_h, const int64_t* pos_start_h,
                            const int32_t* pos_h, const uint8_t* fnorm_h);
int rmu_pgbm25_pop_segments(rmu_pgbm25* h, int n);          /* drops the last n segments */
int rmu_pgbm25_segments(const rmu_pgbm25* h);
int rmu_pgbm25_set_alive(rmu_pgbm25* h, const uint32_t* words_h, int64_t n_words);
/* Q queries; clauses of query q are q_ptr[q] .. q_ptr[q+1], clause c has occur c_occur[c] (0 SHOULD, 1 MUST,
 * 2 MUST_NOT), weight c_weight[c] = (sum of its term idfs) * (1 + K1), and terms ct_term / position offsets ct_off at
 * c_tptr[c] .. c_tptr[c+1] (1..128; the first drives a phrase, so the host puts the rarest first).  cache[256] is the
 * document-length part of the denominator per fieldnorm id.  A row matches when it is alive, matches every MUST
 * clause and no MUST_NOT clause, and (without MUST clauses) at least one SHOULD clause; its score is the float32 sum
 * of weight * (tf / (tf + cache[fieldnorm])) over its matched MUST / SHOULD clauses in clause order (a phrase's tf is
 * its number of occurrences).  out_scores [Q, k] float32 and out_rows [Q, k] int64 global rows, score descending,
 * ties by lower row, -1 padded past the matches.  1 <= k <= 256.  Host buffers; synchronises the stream. */
int rmu_pgbm25_search_host(rmu_pgbm25* h, int Q, const int32_t* q_ptr_h, const int32_t* c_occur_h, const float* c_weight_h,
                           const int32_t* c_tptr_h, const int32_t* ct_term_h, const int32_t* ct_off_h, const float* cache_h,
                           int k, float* out_scores_h, int64_t* out_rows_h, void* stream);

/* ------------------------------------------------------------------ BERT encoder
 * Stands behind HuggingFaceEmbeddings.embed_documents/embed_query (sentence-transformers
 * encode -> BertModel -> Pooling -> Normalize) and HuggingFaceCrossEncoder.score
 * (CrossEncoder.predict -> BertForSequenceClassification). */
/* position_mode: how a token's row of the position table is chosen */
#define RMU_POS_ABSOLUTE 0   /* BERT: the token's offset j in its sequence                                          */
#define RMU_POS_OFFSET 1     /* MPNet, RoBERTa and XLM-RoBERTa (padding index 1): a token of id 1 takes row 1, any
                              * other token row 2 + j - (tokens of id 1 before it); sequences may hold max_pos - 2
                              * tokens (512 for the 514-row tables, 8192 for bge-m3's 8194 rows)                      */

/* The three trailing fields are zero for BERT.  MPNet sets position_mode = RMU_POS_OFFSET and rel_buckets = 32: every
 * attention score gets bias[bucket(key - query), head] of a [32, heads] table shared by all layers (transformers'
 * MPNet relative_position_bucket, 32 buckets, max distance 128).  X-MOD (XLM-R with one language adapter per layer, post-LN,
 * the adapter after the layer's output LayerNorm, which it reuses) sets adapter_dim = A, the bottleneck width: with
 * LN = the layer's output LayerNorm and y = W2 ffn + b2 + x1, the layer's output is LN(D2 gelu(D1 LN(y) + d1) + d2 + LN(y))
 * instead of LN(y).  adapter_dim 0 is no adapter. */
typedef struct rmu_bert_config {
    int32_t vocab_size, hidden, layers, heads, ffn, max_pos, type_vocab, num_labels;
    float ln_eps;
    int32_t position_mode, rel_buckets;
    int32_t adapter_dim;
} rmu_bert_config;

/* What rmu_encoder_create_ex adds, all zero for every model but DeBERTa.  These fields travel in their own struct,
 * not at the end of rmu_bert_config, so that struct keeps its size and layout for callers built against it, and
 * rmu_encoder_create keeps its signature.
 * DeBERTa-v2 / v3 (disentangled attention, share_att_key, pos_att_type c2p | p2c) sets position_buckets = s > 0 and
 * max_relative_positions = the max_position of transformers' make_log_bucket_position (config.max_relative_positions, or
 * max_position_embeddings when that is < 1), with zero position and token-type tables (DeBERTa-v3 adds neither).  With
 * R = LN_rel(rel_embeddings[0:2s]) and, per layer, PQ = Wq R + bq, PK = Wk R + bk split by head like Q and K, every
 * attention score is (Q_i.K_j + Q_i.PK[c] + K_j.PQ[c]) / sqrt(3 d_h), c = clamp(s + bucket(i - j), 0, 2s - 1).
 * Sequences may hold max_pos tokens; d_h must be 64, and rel_buckets and adapter_dim 0.  head_act selects the
 * activation between the pooler and the classifier: RMU_HEAD_TANH (BERT's pooler, 0), RMU_HEAD_GELU (DeBERTa's
 * ContextPooler, erf-GELU) or RMU_HEAD_RELU (DistilBERT's pre_classifier and ReLU; position_buckets must be 0). */
#define RMU_HEAD_TANH 0
#define RMU_HEAD_GELU 1
#define RMU_HEAD_RELU 2
typedef struct rmu_encoder_ext {
    int32_t position_buckets, max_relative_positions, head_act;
} rmu_encoder_ext;

typedef struct rmu_encoder rmu_encoder;

/* weights_h: host fp32 arrays in the canonical order documented in ragmeup_b200/encoder.py
 * (HuggingFace BertModel tensor order; pooler + classifier when has_head; then, when rel_buckets = 32, the relative
 * attention bias [32, heads]; then, when adapter_dim = A > 0, the adapters last, layer by layer: dense1.weight [A, H],
 * dense1.bias [A], dense2.weight [H, A], dense2.bias [H], so every other tensor keeps its index; then, when
 * position_buckets = s > 0, rel_embeddings [2s, H] and LN_rel's weight [H] and bias [H]).  The GEMM weights
 * (query, key, value, attention output, intermediate, output, adapter dense1 and dense2) are held as split fp16 planes,
 * which cannot hold |w| >= 65520: such an element (infinities included) returns RMU_ERR_UNSUPPORTED before any CUDA
 * call.  Embedding tables, biases, LayerNorm parameters and the pooler / classifier stay fp32 and are not limited.  A
 * position_mode other than 0 or 1, a rel_buckets other than 0 or 32, or an adapter_dim that is negative, not a multiple
 * of 128 or larger than ffn returns RMU_ERR_UNSUPPORTED, and a weight count that does not match (the bias table and the
 * adapters included), a null bias table or a null adapter tensor RMU_ERR_ARG, before any CUDA call.  So do, with
 * RMU_ERR_UNSUPPORTED: a head_act other than 0 or 1; position_buckets < 0; position_buckets = 0 with
 * max_relative_positions != 0; position_buckets > 0 with max_relative_positions < s / 2 + 2, s > 4096, d_h != 64,
 * rel_buckets or adapter_dim != 0; and, with RMU_ERR_ARG, a null relative embedding or LN_rel tensor (these for
 * rmu_encoder_create_ex; rmu_encoder_create is rmu_encoder_create_ex with ext = NULL, all zero). */
int rmu_encoder_create(const rmu_bert_config* cfg, const float* const* weights_h, int n_weights, int has_head,
                       rmu_encoder** out);
int rmu_encoder_create_ex(const rmu_bert_config* cfg, const rmu_encoder_ext* ext, const float* const* weights_h,
                          int n_weights, int has_head, rmu_encoder** out);

/* ModernBERT (transformers ModernBertModel / ModernBertForSequenceClassification, model_type "modernbert"): a pre-LN
 * encoder with rotary positions, a GeGLU feed-forward and sliding-window attention on the local layers.  With x the
 * fp32 residual stream:
 *   x = LN_emb(tok_embeddings[id]);  per layer l:  a = (l == 0 ? x : LN_a(x));  x += Wo attn(rope(Wqkv a)) + bo;
 *   x += Wo2 (gelu(Wi_in m + bi_in) * (Wi_gate m + bi_gate)) + bo2 with m = LN_m(x);  hidden = LN_final(x).
 * Wqkv [3H, H] holds q | k | v; q and k are rotated per head (x'[c] = x[c] cos - x[c + d/2] sin, x'[c + d/2] =
 * x[c + d/2] cos + x[c] sin) with the cos / sin of the token's position within its sequence, taken from the global tables
 * on layers with half_window 0 and from the local tables otherwise.  A layer with half_window w > 0 lets query i see key
 * j iff |i - j| <= w.  The head (has_head): logits = classifier(LN_head(gelu(dense(p)))) with p the final hidden state's
 * CLS row or mean over the sequence (`pooling`).  Every GELU is erf-GELU.  Absent biases and LayerNorm shifts are
 * passed as zero arrays.
 *
 * weights_h (host fp32), in this order: tok_embeddings [V, H], embedding norm weight [H], bias [H]; per layer:
 * attn_norm weight [H] and bias [H] (layer 0: not read, may be NULL), Wqkv [3H, H], bqkv [3H], attention Wo [H, H],
 * bo [H], mlp_norm weight [H] and bias [H], Wi [2F, H] (rows 0..F the GELU input, F..2F the gate), bi [2F], mlp Wo
 * [H, F], bo2 [H]; final_norm weight [H] and bias [H]; with has_head: head dense weight [H, H], bias [H], head norm
 * weight [H], bias [H], classifier weight [num_labels, H], bias [num_labels]; then the rope tables cos_global,
 * sin_global, cos_local, sin_local, each [max_pos, d_h / 2] (row p, column i = cos / sin of p * inv_freq[i], as the
 * model computes them in float32).  3 + 12 layers + 2 (+ 6) + 4 tensors.
 * cfg: vocab_size, hidden, layers, heads, ffn (= intermediate_size F), max_pos, num_labels and ln_eps (norm_eps) are
 * read; type_vocab is not (token types are ignored).  Refused before any CUDA call: position_mode, rel_buckets or
 * adapter_dim != 0, d_h other than 32 or 64, hidden not a multiple of 128 or above 1024, F % 64 != 0 and a head_form
 * other than RMU_MB_HEAD_DENSE_GELU_LN (RMU_ERR_UNSUPPORTED); a negative half-window, a pooling other than CLS or mean,
 * rope_rows != max_pos, rope_half != d_h / 2, a wrong tensor count or a null tensor (RMU_ERR_ARG); a GEMM weight with
 * |w| >= 65520 (RMU_ERR_UNSUPPORTED).  Sequences may hold max_pos tokens.  The embed / classify / hidden entry points
 * take such an encoder as any other; every layer runs on every row. */
#define RMU_MB_HEAD_DENSE_GELU_LN 0
typedef struct rmu_modernbert_ext {
    const int32_t* half_window_h;   /* [layers] host: 0 = global attention, w > 0 = sliding window |i - j| <= w */
    int32_t pooling;                /* the classifier's pooling: RMU_POOL_CLS or RMU_POOL_MEAN */
    int32_t head_form;              /* RMU_MB_HEAD_DENSE_GELU_LN */
    int32_t rope_rows, rope_half;   /* shape of each rope table: max_pos, d_h / 2 */
} rmu_modernbert_ext;
int rmu_encoder_create_modernbert(const rmu_bert_config* cfg, const rmu_modernbert_ext* mb, const float* const* weights_h,
                                  int n_weights, int has_head, rmu_encoder** out);

/* Qwen3 (transformers Qwen3Model / Qwen3ForSequenceClassification / Qwen3ForCausalLM, model_type "qwen3"): a decoder
 * run as an encoder, with RMSNorm, grouped-query causal attention, rotary positions and a SwiGLU feed-forward.  With h
 * the fp32 residual stream and RMS(x) = x * rsqrt(mean(x^2) + eps) (the weight multiplies it, not 1 + weight):
 *   h = embed_tokens[id];  per layer:  x = w_in RMS(h);  q = Wq x, k = Wk x, v = Wv x (no biases);
 *   q, k: per head wq_norm RMS(.) / wk_norm RMS(.) over head_dim, then rotate-half rotary at the token's position;
 *   h += Wo attn(q, k, v) with query i seeing keys j <= i of its sequence, query head h reading kv head h / (heads /
 *   kv_heads), scale head_dim^-0.5;  h += Wdown (silu(Wgate x2) * (Wup x2)) with x2 = w_post RMS(h);
 *   hidden = w_norm RMS(h).
 * The outputs take one row per sequence: its last token (embed, RMU_POOL_LAST only, then optionally L2-normalised), or
 * with a head (classify) the rightmost token whose id != pad_token_id (pad_token_id < 0: the last token; no such token:
 * the first), and logits = head [num_labels, H] . hidden(row) (no bias).
 *
 * weights_h (host fp32), in this order: embed_tokens [V, H]; per layer: input_layernorm [H], q_proj [heads d, H],
 * k_proj [kv_heads d, H], v_proj [kv_heads d, H], q_norm [d], k_norm [d], o_proj [H, heads d], post_attention_layernorm
 * [H], gate_proj [F, H], up_proj [F, H], down_proj [H, F]; norm [H]; with has_head: head [num_labels, H]; then the rope
 * tables cos, sin, each [max_pos, d / 2] (row p, column i = cos / sin of p * inv_freq[i] in float32).  1 + 11 layers + 1
 * (+ 1) + 2 tensors.  cfg: vocab_size, hidden, layers, heads, ffn (F), max_pos, num_labels and ln_eps (rms_norm_eps)
 * are read.  Refused before any CUDA call: position_mode, rel_buckets or adapter_dim != 0, head_dim != 128, hidden not a
 * multiple of 128 or above 4096, F % 64 != 0, kv_heads < 1 or heads % kv_heads != 0, and a GEMM weight with |w| >=
 * 65520 (RMU_ERR_UNSUPPORTED); rope_rows != max_pos, rope_half != 64, head_form that disagrees with has_head, a wrong
 * tensor count or a null tensor (RMU_ERR_ARG).
 * Activations enter the GEMMs and attention as split fp16 planes, which cannot hold |x| > 65504: a forward whose
 * normalised rows, q / k / v or SwiGLU outputs leave that range returns RMU_ERR_RANGE and writes no output.  The
 * Qwen3 forward synchronises `stream` to read that flag.  Sequences may hold max_pos tokens. */
#define RMU_QWEN3_HEAD_NONE 0
#define RMU_QWEN3_HEAD_LAST 1
typedef struct rmu_qwen3_ext {
    int32_t kv_heads, head_dim;     /* num_key_value_heads, head_dim (128) */
    int32_t rope_rows, rope_half;   /* shape of each rope table: max_pos, head_dim / 2 */
    int32_t head_form;              /* RMU_QWEN3_HEAD_NONE (has_head 0) or RMU_QWEN3_HEAD_LAST (has_head 1) */
    int32_t pad_token_id;           /* the head's row: the rightmost token whose id differs; < 0: the last token */
} rmu_qwen3_ext;
int rmu_encoder_create_qwen3(const rmu_bert_config* cfg, const rmu_qwen3_ext* ext, const float* const* weights_h,
                             int n_weights, int has_head, rmu_encoder** out);
/* Llama-3 (transformers LlamaModel, model_type "llama"): the Qwen3 decoder above without the per-head q / k RMSNorm.
 * weights_h in Qwen3's order without q_norm and k_norm: embed_tokens; per layer input_layernorm, q_proj, k_proj, v_proj,
 * o_proj, post_attention_layernorm, gate_proj, up_proj, down_proj; norm; rope cos, sin (the caller's table, e.g. with
 * llama3 frequency scaling).  1 + 9 layers + 1 + 2 tensors.  No head: ext->head_form must be RMU_QWEN3_HEAD_NONE.  The
 * shape and weight refusals of rmu_encoder_create_qwen3 apply, before any CUDA call.  rmu_encoder_embed (RMU_POOL_LAST)
 * and rmu_encoder_hidden take it like a Qwen3 embedder. */
int rmu_encoder_create_llama(const rmu_bert_config* cfg, const rmu_qwen3_ext* ext, const float* const* weights_h,
                             int n_weights, rmu_encoder** out);
/* Attention mass of the last layer over token spans of ONE sequence ids [T] (device int32):
 *   out[a][b] = sum over query heads h, rows i in span a, keys j in span b of P_h[i, j]
 * (device float64 [n_spans, n_spans]), P_h the last layer's causal softmax (0 for j > i; query head h reads kv head
 * h / (heads / kv_heads)).  spans [n_spans][2] device int32 (start, end): rows / keys start <= i < end, clamped into
 * [0, T); end <= start is empty; spans may overlap, nest or repeat.  Layers 0..L-2 run as the forward does; the last
 * runs to its q / k step only, and P is never stored.  Each out[a][b] is a float64 sum in a fixed order (the same
 * inputs give the same bits).  Only encoders from rmu_encoder_create_qwen3 without a head or rmu_encoder_create_llama;
 * another encoder, null pointers, T < 1, T > max_pos or n_spans < 1 return RMU_ERR_ARG before any CUDA call; an
 * activation outside the split planes' fp16 range returns RMU_ERR_RANGE and writes nothing.  Synchronises `stream`. */
int rmu_decoder_attention_spans(rmu_encoder* enc, const int32_t* ids, int T, const int32_t* spans, int n_spans,
                                double* out, void* stream);
/* Text generation on a decoder (rmu_encoder_create_qwen3 without a head, or rmu_encoder_create_llama).
 * rmu_decoder_set_lm_head attaches lm_head W_h [vocab_size, hidden] (host fp32; embed_tokens when the embeddings are
 * tied) as split fp16 planes.  Refused before any CUDA call: a null handle or W_h, another kind of encoder, a second
 * call (RMU_ERR_ARG); vocab_size not a multiple of 128 or |w| >= 65520 (RMU_ERR_UNSUPPORTED). */
int rmu_decoder_set_lm_head(rmu_encoder* enc, const float* W_h);
/* NF4 weights for a decoder, as the reference's bitsandbytes load holds them (blocksize 64, fp32 absmax, no double
 * quantisation): each layer's q | k | v, o, gate | up and down projections become packed 4-bit codes [N, K / 2] (the
 * first element in the high nibble) and absmax [N, K / 64], quantised on the device from their hi planes (the fp16
 * cast of the checkpoint's values), and their split planes are freed as the conversion goes, so the handle never holds
 * more device memory than before the call.  The LM head, the embeddings and the norms are unchanged.  Afterwards
 * rmu_decoder_generate and rmu_decoder_attention_spans compute with the dequantised weights fp16(code * absmax): each
 * decode step's projections (M = 1) run a GEMV that reads the codes directly; a prefill dequantises each weight into
 * one scratch plane pair (the size of the largest projection) and runs E1 on it.  Range flag and RMU_ERR_RANGE are as
 * before.  Refused before any CUDA call: a null handle, another kind of encoder, a handle already converted
 * (RMU_ERR_ARG); a projection whose K is not a multiple of 64 or exceeds 49 152 (RMU_ERR_UNSUPPORTED).  A failure
 * part-way leaves a handle that every call refuses; destroy it.  Synchronises the device. */
int rmu_decoder_quantize_nf4(rmu_encoder* enc, void* stream);
/* An NF4 decoder built one layer at a time, so that no layer's weights ever exist on the device in any other form
 * than their codes: Llama (qk_norm 0) or Qwen3 (qk_norm 1), hidden a multiple of 128 up to 8192 (split-plane handles
 * stop at 4096).  rmu_decoder_create_nf4 uploads embed_tokens [vocab_size, hidden], the final norm [hidden] and the
 * rope tables [max_pos, 64] (host fp32), and allocates the prefill's scratch plane pair, the size of the largest
 * projection; the handle has no layers yet.  rmu_decoder_load_layer_nf4 takes layer `layer`'s 9 (Llama) or 11 (Qwen3)
 * host fp32 tensors in rmu_encoder_create_llama's / _qwen3's per-layer order; layers load in order 0, 1, ...  Each
 * projection goes up in chunks of 16 Mi fp32 values (96 MiB of staging with the discarded lo plane, freed when the
 * call returns), becomes its fp16 hi plane in the scratch and is quantised from there: the codes and absmax are bit
 * for bit those of rmu_encoder_create_llama / _qwen3 + rmu_decoder_quantize_nf4 on the same weights, and the device
 * never holds more than the finished handle plus one staging chunk.  Every forward, span, generate and session entry
 * refuses a handle whose layers are not all loaded (RMU_ERR_ARG, naming the missing layer).  Refused before any CUDA
 * call: create_llama's shape refusals with the wider hidden limit, and a projection K not a multiple of 64 or above
 * 49 152 (RMU_ERR_UNSUPPORTED); a layer outside [0, layers) or out of order, a null tensor, a handle not from
 * rmu_decoder_create_nf4 (RMU_ERR_ARG); |w| >= 65520 in a projection (RMU_ERR_UNSUPPORTED, naming the layer and the projection).  A failed
 * load leaves the layer unloaded; the same layer may be loaded again.  load synchronises `stream`. */
int rmu_decoder_create_nf4(const rmu_bert_config* cfg, const rmu_qwen3_ext* ext, int qk_norm, const float* embed_h,
                           const float* final_norm_h, const float* rope_cos_h, const float* rope_sin_h,
                           rmu_encoder** out);
int rmu_decoder_load_layer_nf4(rmu_encoder* enc, int layer, const float* const* tensors_h, void* stream);
/* Token selection, in transformers' order: the repetition penalty (x < 0 ? x * p : x / p) on every id of the prompt and
 * of the generated tokens; then with do_sample 0 the largest logit (the lowest id among equal ones); with do_sample 1
 * x / temperature, top-k (every logit >= the k-th largest survives; 1 <= top_k <= 256, and when more than 256 logits
 * survive through ties at the k-th value, the lowest ids win), top-p over the ascending cumulative softmax (the largest
 * always stays), and an inverse-CDF draw: the first survivor, largest first, whose cumulative weight exceeds u times
 * their total, u a Philox4x32-10 uniform keyed by (seed, step) (no parity with torch.multinomial).  Generation stops
 * after a token in eos_ids[0 .. n_eos) (which is returned), after max_new_tokens, or when prompt and output fill
 * max_pos positions. */
#define RMU_MAX_EOS 8
typedef struct rmu_sampling {
    int32_t do_sample;
    float temperature, top_p, repetition_penalty;   /* repetition_penalty 1: none */
    int32_t top_k;
    int32_t n_eos;
    int32_t eos_ids[RMU_MAX_EOS];
} rmu_sampling;
/* ids_h [T] host int32 prompt -> out_h [max_new_tokens] host int32 generated ids, *n_out of them; logits_h (host,
 * nullable) [max_new_tokens, vocab_size] receives each step's logits before the penalty and sampling.  The prefill writes
 * each layer's rotated k and v into the handle's KV cache (split fp16 planes [kv_heads, T + max_new_tokens, 128] per
 * layer, grown when a call needs more and kept for the next); each step then runs the layers on one row with
 * flash-decoding attention over the cache (fixed-order split merge, no atomics), the final norm, the LM head and the
 * sampler, and synchronises `stream` once to read the token and the fp16 range flag.  Refused before any CUDA call:
 * null pointers, T < 1, max_new_tokens < 1, T >= max_pos, an id outside [0, vocab_size), no LM head, another kind of
 * encoder, n_eos outside 0..8, a repetition_penalty <= 0, and when sampling a temperature <= 0 or top_p outside (0, 1]
 * (RMU_ERR_ARG) or top_k outside 1..256 (RMU_ERR_UNSUPPORTED).  A KV cache that cannot be allocated returns
 * RMU_ERR_CUDA naming the bytes asked for; an activation outside the split planes' fp16 range RMU_ERR_RANGE. */
int rmu_decoder_generate(rmu_encoder* enc, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                         int max_new_tokens, int32_t* out_h, int32_t* n_out, float* logits_h, void* stream);
/* B prompts at once: prompt b = ids_h[cu_h[b] .. cu_h[b + 1]) (host), with seed seeds_h[b] -> out_h [B,
 * max_new_tokens] (row b's first n_out_h[b] entries written, the rest untouched) and logits_h (nullable) [B,
 * max_new_tokens, vocab_size].  Row b is bit for bit what rmu_decoder_generate returns for prompt b and seeds_h[b]:
 * the same tokens and the same logits, on split and NF4 handles, greedy and sampled.  The prompts' longest common
 * prefix (capped so that every prompt keeps one token of its own; none when B = 1) is prefilled once into a shared
 * region of the KV cache, the suffixes as one varlen prefill at their positions after it, and each decode step runs
 * the rows still live at M = live (NF4: one GEMV reads each weight once for all rows), with decode attention over the
 * shared prefix and the row's own keys, the LM head and one sampler CTA per row, and one synchronise of `stream` per
 * step.  Each row stops by rmu_decoder_generate's rules; the call ends when all have stopped.  An activation outside
 * the fp16 range in any row fails the whole call with RMU_ERR_RANGE.  Any failure (a refusal, RMU_ERR_RANGE or a CUDA
 * error) leaves n_out_h[0 .. min(B, 16)) all 0; out_h and logits_h are then unspecified.  Refused before any CUDA call,
 * with rmu_decoder_generate's codes: null pointers, B < 1 or B > RMU_MAX_GENERATE_BATCH, an empty prompt,
 * max_new_tokens < 1, no LM head, another kind of encoder, a broken NF4 handle, a prompt of >= max_pos tokens, the
 * sampling settings rmu_decoder_generate refuses, an id outside [0, vocab_size). */
#define RMU_MAX_GENERATE_BATCH 16
int rmu_decoder_generate_batch(rmu_encoder* enc, const int32_t* ids_h, const int32_t* cu_h, int B, const rmu_sampling* s,
                               const uint64_t* seeds_h, int max_new_tokens, int32_t* out_h, int32_t* n_out_h,
                               float* logits_h, void* stream);
/* Prompt-lookup decoding (transformers' prompt_lookup_num_tokens): rmu_decoder_generate's tokens and logits, bit for
 * bit, on split and NF4 handles, greedy and sampled, with fewer model passes when the reply copies the prompt.  After
 * the prefill each pass feeds the pending token plus k drafts (k = min(lookup_tokens, 15), further capped so that no
 * pass reaches past max_new_tokens or max_pos; 15 because a pass runs at most RMU_MAX_GENERATE_BATCH rows): the
 * continuation of the first earlier match of the sequence's last n-gram (rmu_prompt_lookup_draft over the prompt and
 * the tokens so far, max_length T + max_new_tokens).  The k + 1 rows run as one batched decode step whose row j
 * computes exactly the sequential step's logits and samples with that step's penalty bits and Philox uniform; the
 * host keeps row 0's token and row j's while row j - 1's token equals draft j.  logits_h receives the kept rows only.
 * lookup_tokens 0 runs rmu_decoder_generate's steps.  A pass that raises the fp16 range flag is redone as a single-row
 * step, and RMU_ERR_RANGE is returned only if that step raises it too.  n_passes (host, nullable) <- the model passes
 * after the prefill.  Refused before any CUDA call as rmu_decoder_generate refuses, and lookup_tokens < 0 or
 * max_ngram < 1 (RMU_ERR_ARG). */
int rmu_decoder_generate_lookup(rmu_encoder* enc, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                                int max_new_tokens, int lookup_tokens, int max_ngram, int32_t* out_h, int32_t* n_out,
                                float* logits_h, int32_t* n_passes, void* stream);
/* The prompt-lookup drafter (host only, no CUDA call), as transformers' PromptLookupCandidateGenerator.get_candidates
 * proposes without a logits processor or eos ids: for n-gram sizes g = min(max_ngram, n - 1) down to 1, the first
 * position i (left to right) where ids[i .. i + g) equals the last g ids and ids[i + g .. min(i + g + k, n, max_len))
 * is not empty; that continuation goes to out and its length is returned.  0 when nothing matches or max_len == n + 1.
 * Null pointers, n < 1, k < 1 or max_ngram < 1 return RMU_ERR_ARG. */
int rmu_prompt_lookup_draft(const int32_t* ids, int n, int k, int max_ngram, int max_len, int32_t* out);
/* Speculative decoding with a draft model (transformers' assistant_model): rmu_decoder_generate's tokens and logits on
 * enc, bit for bit, on any mix of split and NF4 handles, greedy and sampled, whatever the draft computes.  The draft
 * is another decoder handle with an LM head and the same vocab_size.  Passes run as in rmu_decoder_generate_lookup,
 * with k drafts from the draft model: its own prefill of the prompt into its own KV cache on the first pass, then per
 * pass the rows its cache lacks (1 or 2 in steady state) and k - 1 single-row steps, each feeding the draft before it
 * on the device, with one synchronise per pass.  Draft j samples with the target's settings, the presence bits of the
 * tokens so far plus drafts 1 .. j - 1, and the Philox uniform of the output index it stands for, so a draft that
 * computes the target's logits has every draft kept.  k starts at min(num_tokens, 15) and is capped as in
 * rmu_decoder_generate_lookup and so that no draft position reaches the draft's max_pos; RMU_ASSIST_HEURISTIC then
 * adds 2 after a pass that kept every draft and subtracts 1 (to at least 1) after any other, within this call.
 * num_tokens 0 runs rmu_decoder_generate's steps.  A draft pass that raises the draft's fp16 range flag clears it and
 * proposes no drafts; it never fails the call.  n_passes (target passes after the prefill), n_drafted (drafts
 * proposed) and n_kept (drafts emitted as tokens) are host and nullable; logits_h receives the target's logits only.
 * Both handles are held for the whole call.  Refused before any CUDA call as rmu_decoder_generate refuses, and: a null
 * draft, the target as its own draft, num_tokens < 0 or another schedule (RMU_ERR_ARG); a draft that is not a decoder,
 * has no LM head or is an incomplete NF4 handle, a vocab_size that differs from the target's, or a draft on another
 * device (RMU_ERR_ARG). */
#define RMU_ASSIST_CONSTANT 0    /* transformers' num_assistant_tokens_schedule "constant" */
#define RMU_ASSIST_HEURISTIC 1   /* "heuristic" / "heuristic_transient": +2 after a fully kept pass, else -1 (min 1) */
int rmu_decoder_generate_assisted(rmu_encoder* enc, rmu_encoder* draft, const int32_t* ids_h, int T,
                                  const rmu_sampling* s, uint64_t seed, int max_new_tokens, int num_tokens,
                                  int schedule, int32_t* out_h, int32_t* n_out, float* logits_h, int32_t* n_passes,
                                  int32_t* n_drafted, int32_t* n_kept, void* stream);
/* Continuous batching: a decode session of one decoder handle (with an LM head) that outlives a call.  Requests join
 * it (rmu_decoder_session_add) and leave it (when they stop, or rmu_decoder_session_cancel) between steps; each
 * rmu_decoder_session_step runs one decode step over every live row at M = live (at most RMU_MAX_GENERATE_BATCH).
 * Each request's tokens and logits are bit for bit what rmu_decoder_generate returns for its prompt, settings, seed and
 * max_new_tokens, on split and NF4 handles, whenever it joins and whatever rows share its steps.
 *
 * The session owns its KV cache (the handle cache's layout; rmu_decoder_generate[_batch|_lookup] never touch it): a
 * request of T prompt tokens holds the rows [base, base + min(T + max_new_tokens, max_pos)), placed first fit among the
 * free gaps; when none fits the cache grows (one 2D copy to the new pitch, so no live row moves).  Every entry point
 * holds the handle's lock for its own duration only, so other calls on the handle run between steps.  Calls may come
 * from different threads on different streams: each waits on the session's last use and on the handle's workspace.
 *
 * rmu_decoder_session_create / _destroy: a handle's sessions are destroyed before the handle; destroy waits for the
 * session's last use.  Refused: a null pointer or another kind of encoder (RMU_ERR_ARG). */
typedef struct rmu_gen_session rmu_gen_session;
int rmu_decoder_session_create(rmu_encoder* enc, rmu_gen_session** out);
void rmu_decoder_session_destroy(rmu_gen_session* s);
/* A row's status after a token: RMU_GEN_LIVE, or why it stopped (the row is then released in the same call), or a
 * negative error code (RMU_ERR_RANGE: this request's own activations left the fp16 range; no token). */
#define RMU_GEN_LIVE 0
#define RMU_GEN_EOS 1
#define RMU_GEN_MAX_NEW 2
#define RMU_GEN_MAX_POS 3
/* Admit B requests (1 .. RMU_MAX_GENERATE_BATCH): prompt b = ids_h[cu_h[b] .. cu_h[b + 1]) with settings s_h[b], seed
 * seeds_h[b] and max_new_h[b] (all host).  They are prefilled together as one varlen run into their own regions (an
 * NF4 handle's one-token prompts alone, on the decode GEMV), and each samples its first token: slot_h[b] <- its row
 * (-1 when it stopped or failed), tok_h[b], status_h[b]; logits_h (host, nullable) [B, vocab_size] <- each first
 * token's logits.  When the range flag rises the requests are redone one at a time, and only those whose own run
 * raises it end with RMU_ERR_RANGE.  Refused before any CUDA call with rmu_decoder_generate's codes (null pointers,
 * an empty prompt, max_new < 1, T >= max_pos, an id out of range, the sampling settings rmu_decoder_generate refuses,
 * no LM head, a broken NF4 handle).  RMU_ERR_BUSY, with the session unchanged: fewer than B free rows, or a KV cache
 * that cannot grow while rows are live (with no live row that failure is RMU_ERR_CUDA naming the positions).  Any
 * other failure releases the call's new rows.  Synchronises `stream`. */
int rmu_decoder_session_add(rmu_gen_session* s, const int32_t* ids_h, const int32_t* cu_h, int B, const rmu_sampling* s_h,
                            const uint64_t* seeds_h, const int32_t* max_new_h, int32_t* slot_h, int32_t* tok_h,
                            int32_t* status_h, float* logits_h, void* stream);
/* One decode step over every live row, in slot order: *n_h <- the rows (0 when none is live: no CUDA call), row r ->
 * slot_h[r], tok_h[r], status_h[r] and logits_h (host, nullable) [16, vocab_size] row r.  A range error is handled as
 * in rmu_decoder_session_add.  A failed step (a CUDA error, an allocation that fails) releases every live row and
 * reports none.  Synchronises `stream`. */
int rmu_decoder_session_step(rmu_gen_session* s, int32_t* slot_h, int32_t* tok_h, int32_t* status_h, int32_t* n_h,
                             float* logits_h, void* stream);
/* Release a live row without output; a slot that is not live returns RMU_ERR_ARG.  No CUDA call. */
int rmu_decoder_session_cancel(rmu_gen_session* s, int slot);
/* The live rows, the KV cache's capacity in positions and live_mask (nullable): bit i set when slot i is live.  No
 * CUDA call. */
int rmu_decoder_session_info(rmu_gen_session* s, int32_t* live, int32_t* cap_positions, uint32_t* live_mask);
void rmu_encoder_destroy(rmu_encoder* enc);

#define RMU_POOL_MEAN 0
#define RMU_POOL_CLS 1
#define RMU_POOL_LAST 2   /* each sequence's last token: Qwen3 encoders only, which accept no other pooling */

/* ragged batch: ids/type_ids [total_tokens] int32, cu_seqlens [B+1] int32 (all device); type_ids may be null (all 0).
 * max_seqlen must be at least the longest sequence in cu_seqlens; only max_seqlen itself is checked against
 * max_position_embeddings (max_seqlen + 2 <= max_pos with RMU_POS_OFFSET; cu_seqlens is on the device).  Out-of-range
 * inputs are clamped on the device, where
 * HuggingFace raises an IndexError: token ids into [0, vocab_size), type ids into [0, type_vocab), and positions past
 * max_position_embeddings - 1 take that last row.  An empty sequence (cu_seqlens[b + 1] == cu_seqlens[b]) is allowed,
 * but a batch must hold at least one token: B < 1 or total_tokens < 1 (a batch of empty sequences only) returns
 * RMU_ERR_ARG before any CUDA call.  B has no upper limit besides int and device memory (attention runs batches of more
 * than 65 535 sequences in slices).  These rules hold for every rmu_encoder_* entry point below.
 * out [B, hidden] fp32 sentence embeddings; an empty sequence gets a zero vector. */
int rmu_encoder_embed(rmu_encoder* enc, const int32_t* ids, const int32_t* type_ids, const int32_t* cu_seqlens,
                      int B, int total_tokens, int max_seqlen, int pool_mode, int normalize, float* out,
                      void* stream);
/* cross-encoder logits: out [B, num_labels] fp32 (raw logits; activation is the caller's).  An empty sequence has a
 * zero CLS hidden state: its logits are W_c tanh(b_p) + b_c. */
int rmu_encoder_classify(rmu_encoder* enc, const int32_t* ids, const int32_t* type_ids, const int32_t* cu_seqlens,
                         int B, int total_tokens, int max_seqlen, float* out, void* stream);
/* last hidden state [total_tokens, hidden] fp32 (tests / provenance) */
int rmu_encoder_hidden(rmu_encoder* enc, const int32_t* ids, const int32_t* type_ids, const int32_t* cu_seqlens,
                       int B, int total_tokens, int max_seqlen, float* out, void* stream);
/* host-buffer variants (H2D of the token batch + D2H of the result inside; synchronise) */
int rmu_encoder_embed_host(rmu_encoder* enc, const int32_t* ids_h, const int32_t* type_ids_h,
                           const int32_t* cu_seqlens_h, int B, int total_tokens, int max_seqlen, int pool_mode,
                           int normalize, float* out_h, void* stream);
int rmu_encoder_classify_host(rmu_encoder* enc, const int32_t* ids_h, const int32_t* type_ids_h,
                              const int32_t* cu_seqlens_h, int B, int total_tokens, int max_seqlen, float* out_h,
                              void* stream);

/* sentence-transformers Dense modules after Pooling (distiluse-base-multilingual-cased-v2, LaBSE): attaches the chain
 * y_{l+1} = act_l(W_l y_l + b_l), l = 0..n_layers-1, with y_0 the pooled row [dims[0] = hidden], W_l [dims[l+1], dims[l]]
 * and b_l [dims[l+1]] host fp32 (b_h or any b_h[l] may be NULL: no bias), act_l RMU_DENSE_IDENTITY or RMU_DENSE_TANH.
 * Afterwards rmu_encoder_embed and rmu_encoder_embed_host pool without normalising, run the chain in fp32 (one fmaf
 * chain per output, fixed order, no atomics) and then, when normalize, apply Normalize: they write [B, dims[n_layers]].
 * rmu_encoder_hidden and rmu_encoder_classify are unchanged.  Refused: a null handle, dims, W_h or acts, n_layers <= 0,
 * dims[0] != hidden, a width <= 0, a null W_h[l], or a second call (RMU_ERR_ARG); an act other than 0 or 1, or a
 * Qwen3 / Llama handle (RMU_ERR_UNSUPPORTED). */
#define RMU_DENSE_IDENTITY 0
#define RMU_DENSE_TANH 1
int rmu_encoder_set_dense(rmu_encoder* enc, int n_layers, const int32_t* dims, const float* const* W_h,
                          const float* const* b_h, const int32_t* acts);

/* ------------------------------------------------------------------ ColBERT late interaction
 * Stands behind HuggingFaceCrossEncoder.score on a ColBERT checkpoint (the reference README's `rerank_model`
 * colbert-ir/colbertv2.0): every query and document token gets a unit vector, linear(h) / max(||linear(h)||, 1e-12)
 * of the last hidden state h, and a (query, document) pair scores sum over the query's tokens of the maximum dot product
 * with the document's kept tokens (MaxSim).
 *
 * cfg and weights_h as rmu_encoder_create with has_head = 0 (an X-MOD backbone, colbert-xm, brings its adapters at
 * the end of weights_h and gets rmu_encoder_create's adapter_dim checks and error codes); linear_h [dim, hidden] host fp32 (ColBERT's `linear`, no
 * bias), held as split fp16 planes like the GEMM weights: |w| >= 65520 returns RMU_ERR_UNSUPPORTED before any CUDA call,
 * as does a dim above 128 that is not a multiple of 128, or rel_buckets != 0.  Token ids only: ColBERT sends no token
 * types. */
typedef struct rmu_colbert rmu_colbert;
int rmu_colbert_create(const rmu_bert_config* cfg, const float* const* weights_h, int n_weights, const float* linear_h,
                       int dim, rmu_colbert** out);
void rmu_colbert_destroy(rmu_colbert* cb);
int rmu_colbert_dim(const rmu_colbert* cb);
/* token vectors of a ragged batch (the rules of rmu_encoder_embed) -> out [total_tokens, dim] fp32.  nkeys [B] int32
 * (nullable): the attention keys of sequence b are its first min(max(nkeys[b], 1), S_b) tokens in every layer, while
 * every token is a query row (ColBERT's [MASK] query padding, attend_to_mask_tokens = false).  keep [total_tokens] uint8
 * (nullable = all kept): a token with keep 0 gets a zero vector.  All device pointers. */
int rmu_colbert_vectors(rmu_colbert* cb, const int32_t* ids, const int32_t* cu_seqlens, const int32_t* nkeys,
                        const uint8_t* keep, int B, int total_tokens, int max_seqlen, float* out, void* stream);
/* MaxSim: q [*, dim] query token vectors with q_cu, d [*, dim] document token vectors with d_cu and d_keep (nullable =
 * all kept; a token with keep 0 is skipped, never a candidate for the maximum); pair p scores query pair_q[p] against
 * document pair_d[p] -> out [n_pairs] fp32.  Each pair is computed in a fixed order from its own token lists, so its
 * score does not depend on the other pairs of the call.  A document without a kept token scores -inf.  Indices must be
 * in range (device arrays, not checked); n_pairs = 0 launches nothing.  All device pointers. */
int rmu_colbert_maxsim(const float* q, const int32_t* q_cu, const float* d, const int32_t* d_cu, const uint8_t* d_keep,
                       int dim, const int32_t* pair_q, const int32_t* pair_d, int n_pairs, float* out, void* stream);
/* the whole score from HOST buffers: the query batch (q_nkeys_h nullable) in one run, the documents in runs of at most
 * max_tokens_per_batch tokens (a longer document runs alone), then MaxSim over the pairs -> out_h [n_pairs].  Pair
 * indices out of range, cu arrays that do not start at 0, end at the token count or decrease, and a document without a
 * kept token return RMU_ERR_ARG before any CUDA call.  Synchronises `stream`. */
int rmu_colbert_score_host(rmu_colbert* cb, const int32_t* q_ids_h, const int32_t* q_cu_h, const int32_t* q_nkeys_h, int nq,
                           int q_tokens, const int32_t* d_ids_h, const int32_t* d_cu_h, const uint8_t* d_keep_h, int nd,
                           int d_tokens, const int32_t* pair_q_h, const int32_t* pair_d_h, int n_pairs,
                           int max_tokens_per_batch, float* out_h, void* stream);

/* ------------------------------------------------------------------ kernel-level test entry points,
 * not part of the product path.  Each runs ONE encoder kernel through the launcher the encoder itself uses, on
 * split fp16 planes the caller owns (v = hi + lo, hi = fp16(v), lo = fp16(v - hi); planes are fp16 bit patterns,
 * row-major, device pointers); they allocate nothing.  Shapes the kernels do not take return RMU_ERR_UNSUPPORTED
 * before any CUDA call.  For tests that compare each kernel with a high-precision reference. */
#define RMU_GEMM_BIAS_F32 0           /* out_f32 = A W^T + bias                                         */
#define RMU_GEMM_BIAS_GELU_SPLIT 1    /* out planes = split(gelu_erf(A W^T + bias))                     */
#define RMU_GEMM_BIAS_RESID_F32 2     /* out_f32 = A W^T + bias + (res_hi + res_lo)                     */
#define RMU_GEMM_BIAS_SPLIT_QSCALE 3  /* out planes = split((A W^T + bias) * (col < qcols ? qscale : 1)) */
#define RMU_GEMM_BIAS_SPLIT_ROPE 4    /* mode 3 with columns < 2 qcols (q, k) rotated per head at pos[row]      */
#define RMU_GEMM_BIAS_GEGLU_SPLIT 5   /* W in 128-row blocks of 64 input | 64 gate rows: out planes [M, N / 2] =
                                       * split(gelu_erf(in + b_in) * (gate + b_gate))                           */
#define RMU_GEMM_BIAS_RESF32_F32 6    /* out_f32 = A W^T + bias + res_f32 (res_f32 may equal out_f32)            */
#define RMU_GEMM_BIAS_SWIGLU_SPLIT 7  /* W blocked as mode 5: out planes [M, N / 2] = split(silu(in + b_in) *
                                       * (gate + b_gate)), silu(g) = g / (1 + exp(-g))                          */

/* For tests: E1 on A [a_rows, K] (rows M..a_rows are read by the TMA loads but never reach the output) and
 * W [N, K]; bias [N], res [M, N], out [M, N].  N % 128 == 0, K % 64 == 0, a_rows >= M.  max_ctas caps the
 * persistent grid (0 = the device's SM count), so a small problem can put many tiles through one CTA. */
int rmu_debug_gemm(int mode, const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                   const uint16_t* w_lo, int M, int N, int K, const float* bias, const uint16_t* res_hi,
                   const uint16_t* res_lo, int qcols, float qscale, int max_ctas, float* out_f32, uint16_t* out_hi,
                   uint16_t* out_lo, void* stream);
/* For tests: E1 in the ModernBERT modes 4, 5 and 6, shapes as rmu_debug_gemm.  Mode 4: pos [M] int32 (device) is each
 * row's position, clamped into the rope_cos / rope_sin tables [rope_rows, head_dim / 2] (device fp32); qcols (= H) is a
 * multiple of 64 and of head_dim (32 or 64); out planes [M, N].  Mode 5: W as the mode describes it, out planes
 * [M, N / 2].  Mode 6: res_f32 [M, N], out_f32 [M, N], which may be the same array.  Another mode returns RMU_ERR_ARG. */
int rmu_debug_gemm_ex(int mode, const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                      const uint16_t* w_lo, int M, int N, int K, const float* bias, const float* res_f32, int qcols,
                      float qscale, const int32_t* pos, const float* rope_cos, const float* rope_sin, int rope_rows,
                      int head_dim, int max_ctas, float* out_f32, uint16_t* out_hi, uint16_t* out_lo, void* stream);
/* For tests: E2 with ModernBERT's sliding window, as a local layer runs it: key j is visible to query i iff
 * |i - j| <= window (window > 0), 10 warps, every query row; otherwise as rmu_debug_attention.  With window >= the
 * longest sequence - 1 the output equals rmu_debug_attention's bit for bit. */
int rmu_debug_attention_window(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu_seqlens, int B, int H,
                               int heads, int max_seqlen, int window, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* For tests: ModernBERT's head on pooled rows [B, H] (device fp32): out [B, num_labels] = cw LN(gelu_erf(dense_w p +
 * dense_b)) + cb, LN with norm_w, norm_b and eps.  1 <= H <= 1024. */
int rmu_debug_modernbert_head(const float* pooled, int B, int H, int num_labels, const float* dense_w, const float* dense_b,
                              const float* norm_w, const float* norm_b, float eps, const float* cw, const float* cb,
                              float* out, void* stream);
/* For tests: E1 in mode 7 (SwiGLU), shapes as rmu_debug_gemm, out planes [M, N / 2].  range_flag (device int32, may be
 * NULL) is set to 1 when an output of rows 0..M has |x| > 65504 or is NaN; it is never cleared. */
int rmu_debug_gemm_swiglu(const uint16_t* a_hi, const uint16_t* a_lo, int64_t a_rows, const uint16_t* w_hi,
                          const uint16_t* w_lo, int M, int N, int K, const float* bias, int max_ctas, uint16_t* out_hi,
                          uint16_t* out_lo, int32_t* range_flag, void* stream);
/* For tests: Qwen3's RMSNorm of T fp32 rows [T, H] (device) -> split planes [T, H] = split(w * (x * rsqrt(mean(x^2) +
 * eps))).  H a multiple of 128 up to 8192 (256 threads per row above 4096).  range_flag (device, may be NULL) as
 * rmu_debug_gemm_swiglu's. */
int rmu_debug_rmsnorm(const float* x, int T, int H, const float* w, float eps, uint16_t* hi, uint16_t* lo,
                      int32_t* range_flag, void* stream);
/* For tests: Qwen3's q / k step on the fp32 QKV rows [T, (heads + 2 kv_heads) 128] (q | k | v, heads of 128): per
 * token and q or k head, RMSNorm over the head with q_norm / k_norm [128], rotate-half rotary at pos[t] (clamped into
 * the cos / sin tables [rope_rows, 64]), q times qscale; v unchanged; all written as split planes of the same shape.
 * q_norm and k_norm both NULL: Llama's step, the same without the RMSNorm; exactly one NULL returns RMU_ERR_ARG.
 * range_flag as above. */
int rmu_debug_qk_norm_rope(const float* qkv, int T, int heads, int kv_heads, const int32_t* pos, const float* q_norm,
                           const float* k_norm, float eps, float qscale, const float* rope_cos, const float* rope_sin,
                           int rope_rows, uint16_t* hi, uint16_t* lo, int32_t* range_flag, void* stream);
/* For tests: Qwen3's causal grouped-query attention on the planes [T, (heads + 2 kv_heads) 128] of a ragged batch (q
 * pre-scaled by log2(e) / sqrt(128)), cu_seqlens [B+1] -> ctx planes [T, heads 128].  Query i of a sequence sees its
 * keys j <= i; query head h reads kv head h / (heads / kv_heads).  heads % kv_heads != 0 returns RMU_ERR_UNSUPPORTED. */
int rmu_debug_attention_causal(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu_seqlens, int B,
                               int heads, int kv_heads, int max_seqlen, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* For tests: the span attention of rmu_decoder_attention_spans on given planes [T, (heads + 2 kv_heads) 128] of one
 * sequence (q pre-scaled by log2(e) / sqrt(128), as the q / k step leaves it) -> out [n_spans, n_spans] float64, spans as
 * there.  Allocates its workspace stream-ordered on `stream`.  Null pointers, T, heads, kv_heads or n_spans < 1 return
 * RMU_ERR_ARG, heads % kv_heads != 0 RMU_ERR_UNSUPPORTED, before any CUDA call. */
int rmu_debug_attention_spans(const uint16_t* qkv_hi, const uint16_t* qkv_lo, int T, int heads, int kv_heads,
                              const int32_t* spans, int n_spans, double* out, void* stream);
/* For tests: Qwen3's output rows on fp32 residual rows x [T, H] (device): per sequence b the row cu[b + 1] - 1
 * (pad_id < 0) or the rightmost row whose ids[] != pad_id (none: the first row), y = w RMS(x_row); then out [B, H] = y
 * (optionally L2-normalised) when head is NULL, else out [B, num_labels] = head [num_labels, H] . y.  An empty sequence
 * gives zeros.  H a multiple of 128 up to 4096. */
int rmu_debug_last_token(const float* x, const int32_t* ids, const int32_t* cu_seqlens, int B, int H, const float* w,
                         float eps, int pad_id, int normalize, const float* head, int num_labels, float* out, void* stream);
/* For tests: E2 on the QKV planes [T, 3H] of a ragged batch (q | k | v, q pre-scaled by log2(e) / sqrt(d_h) as the
 * QKV epilogue leaves it), cu_seqlens [B+1] int32 -> ctx planes [T, H].  d_h = H / heads is 32 or 64; warps must be
 * 10 (160 query rows per CTA), any other value returns RMU_ERR_ARG. */
int rmu_debug_attention(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu_seqlens, int B, int H,
                        int heads, int max_seqlen, int warps, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* For tests: E2 with a key limit per sequence, as rmu_colbert_vectors runs it: nkeys [B] int32 on the device, sequence
 * b's keys are its first min(max(nkeys[b], 1), S_b) rows and every row is a query.  warps as rmu_debug_attention. */
int rmu_debug_attention_keys(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu_seqlens, const int32_t* nkeys,
                             int B, int H, int heads, int max_seqlen, int warps, uint16_t* ctx_hi, uint16_t* ctx_lo,
                             void* stream);
/* For tests: E3 ln_kernel, LayerNorm of pre [T, H] fp32 (biased variance, eps inside the sqrt) -> planes [T, H].
 * H % 128 == 0, H <= 1024. */
int rmu_debug_layernorm(const float* pre, int T, int H, const float* gamma, const float* beta, float eps,
                        uint16_t* out_hi, uint16_t* out_lo, void* stream);
/* For tests: E3 embed_ln_kernel on fp32 tables word [vocab, H], pos [max_pos, H], typ [type_vocab, H], ids / type_ids
 * [T] int32 (type_ids null = all 0) and cu_seqlens [B+1] -> LayerNorm(word + typ + pos) planes [T, H], clamping ids,
 * type ids and positions as rmu_encoder_embed does.  H % 128 == 0, H <= 1024; null pointers (but type_ids) and B, T,
 * vocab, max_pos or type_vocab < 1 return RMU_ERR_ARG. */
int rmu_debug_embed_ln(const int32_t* ids, const int32_t* type_ids, const int32_t* cu_seqlens, int B, int T, int H,
                       int vocab, int max_pos, int type_vocab, const float* word, const float* pos, const float* typ,
                       const float* gamma, const float* beta, float eps, uint16_t* out_hi, uint16_t* out_lo, void* stream);
/* For tests: the same with the position rule pos_mode (RMU_POS_ABSOLUTE is rmu_debug_embed_ln; RMU_POS_OFFSET compares
 * the raw ids with 1, then clamps positions to max_pos - 1).  Another pos_mode returns RMU_ERR_ARG. */
int rmu_debug_embed_ln_pos(const int32_t* ids, const int32_t* type_ids, const int32_t* cu_seqlens, int B, int T, int H,
                           int vocab, int max_pos, int type_vocab, const float* word, const float* pos, const float* typ,
                           const float* gamma, const float* beta, float eps, int pos_mode, uint16_t* out_hi,
                           uint16_t* out_lo, void* stream);
/* Host only, no GPU work: the attention bias table rmu_encoder_create builds from bias_h [buckets, heads] fp32 ->
 * table_h [heads, 255] fp32, entry (h, r + 127) = bias_h[bucket(r), h] * log2(e) for r = key - query in [-127, 127]
 * (every |r| >= 127 falls in the last bucket of its side).  buckets other than 32 return RMU_ERR_UNSUPPORTED. */
int rmu_relative_bias_table(const float* bias_h, int buckets, int heads, float* table_h);
/* For tests: E2 with the relative bias, rel_table [heads, 255] fp32 on the device (rmu_relative_bias_table's layout),
 * 10 warps.  cls_q_hi / cls_q_lo null: every query row, ctx [T, H]; non-null: the compact Q planes [B, H] of query row 0
 * of each sequence (the last layer's CLS-only mode), ctx [B, H]. */
int rmu_debug_attention_bias(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const uint16_t* cls_q_hi,
                             const uint16_t* cls_q_lo, const int32_t* cu_seqlens, int B, int H, int heads, int max_seqlen,
                             const float* rel_table, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* Host only, no GPU work: DeBERTa's relative position buckets, out_h[r + n - 1] = make_log_bucket_position(r,
 * buckets, max_position) for r in [-(n - 1), n - 1], in torch's float32 arithmetic, as rmu_encoder_create builds them.
 * buckets < 2, max_position < buckets / 2 + 2 or n < 1 return RMU_ERR_UNSUPPORTED / RMU_ERR_ARG. */
int rmu_log_bucket_table(int buckets, int max_position, int n, int32_t* out_h);
/* For tests: E2 with DeBERTa's disentangled position terms, as the encoder runs it: the terms C2P (query rows against
 * PK) and P2C (every key against PQ') into ws, then E2 adding C2P[i, c] + P2C[j, c] to each score.  qkv planes [T, 3H]
 * with q pre-scaled by log2(e) / sqrt(3 d_h); pos planes [2s, 2H] = PQ' | PK, PQ' pre-scaled like q; cidx_h (HOST)
 * [2 max_seqlen - 1] int32, entry r + max_seqlen - 1 = clamp(s + bucket(r), 0, 2s - 1), non-decreasing in r; it is
 * copied into the tail of ws.  cls_q null: every query row, ctx [T, H]; non-null: the compact Q planes [B, H] of query
 * row 0 of each sequence, ctx [B, H].  ws (device fp32) holds (qrows + T) heads W + 2 max_seqlen - 1 elements, qrows = B
 * (CLS) or T and W = cidx_h[last] - cidx_h[0] + 1.  d_h must be 64; a smaller ws, a cidx_h that decreases, is negative
 * or reaches row 2 position_buckets of the pos planes, null pointers or bad sizes return RMU_ERR_ARG before any CUDA
 * call. */
int rmu_debug_attention_disentangled(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const uint16_t* cls_q_hi,
                                     const uint16_t* cls_q_lo, const int32_t* cu_seqlens, int B, int T, int H, int heads,
                                     int max_seqlen, const uint16_t* pos_hi, const uint16_t* pos_lo, int position_buckets,
                                     const int32_t* cidx_h, float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo,
                                     void* stream);
/* For tests: E4 pool_kernel, RMU_POOL_MEAN or RMU_POOL_CLS of planes [T, H] per sequence of cu_seqlens [B+1], then
 * x / max(||x||, 1e-12) when normalize -> out [B, H] fp32 (an empty sequence gives zeros).  1 <= H <= 1024. */
int rmu_debug_pool(const uint16_t* hi, const uint16_t* lo, const int32_t* cu_seqlens, int B, int H, int pool_mode,
                   int normalize, float* out, void* stream);
/* For tests: E4 cls_head_kernel on planes [T, H] and cu_seqlens [B+1] (h_cls = row cu_seqlens[b], 0 for an empty
 * sequence), pooler pw [H, H] / pb [H], classifier cw [num_labels, H] / cb [num_labels] fp32 -> out [B, num_labels]
 * = cw tanh(pw h_cls + pb) + cb.  1 <= H <= 1024. */
int rmu_debug_cls_head(const uint16_t* hi, const uint16_t* lo, const int32_t* cu_seqlens, int B, int H, int num_labels,
                       const float* pw, const float* pb, const float* cw, const float* cb, float* out, void* stream);
/* For tests: copies layer `layer`'s PQ' | PK planes [2s, 2H] of a DeBERTa encoder (position_buckets = s > 0), as
 * rmu_encoder_create_ex computed them, into hi / lo (device, 2s * 2H fp16 each).  Another encoder or layer returns
 * RMU_ERR_ARG. */
int rmu_debug_encoder_position_planes(const rmu_encoder* enc, int layer, uint16_t* hi, uint16_t* lo, void* stream);
/* For tests: the same with the activation between pooler and classifier, head_act RMU_HEAD_TANH (rmu_debug_cls_head) or
 * RMU_HEAD_GELU (DeBERTa's ContextPooler, erf-GELU), as rmu_encoder_create_ex's ext->head_act selects it.  Another
 * head_act returns RMU_ERR_ARG. */
int rmu_debug_cls_head_act(const uint16_t* hi, const uint16_t* lo, const int32_t* cu_seqlens, int B, int H, int num_labels,
                           const float* pw, const float* pb, const float* cw, const float* cb, int head_act, float* out,
                           void* stream);
/* For tests: n fp32 values -> (hi, lo) planes, as every GEMM weight is uploaded; and hi + lo -> n fp32 values, as
 * rmu_encoder_hidden returns the last hidden state.  n < 0 or a null pointer return RMU_ERR_ARG; n = 0 launches
 * nothing. */
/* For tests: one Dense module on device rows x [B, n_in] fp32: y [B, n_out] = act(W x + b) with W [n_out, n_in], b
 * [n_out] or NULL, act RMU_DENSE_IDENTITY or RMU_DENSE_TANH, then y / max(||y||, 1e-12) per row when normalize, as
 * rmu_encoder_set_dense's chain runs it.  A null pointer or a width or B <= 0 returns RMU_ERR_ARG, another act
 * RMU_ERR_UNSUPPORTED. */
int rmu_debug_dense(const float* x, int B, int n_in, int n_out, const float* W, const float* b, int act, int normalize,
                    float* y, void* stream);
/* For tests: the batched decode's attention.  Row b's q sits qld halves after row b - 1's ([heads 128] each); it reads
 * keys [0, pos_h[b] + 1) of the cache kv, key k at row k when k < P, else k + shift_h[b] (pos_h, shift_h host int32
 * [B]) -> ctx [B, heads 128].  Row b equals rmu_debug_attention_decode on a cache holding those keys at rows 0 ..
 * pos_h[b].  ws holds B * heads * ceil(n / 64) * 130 + 2 B floats, n the largest pos_h + 1.  Null pointers, B outside
 * 1 .. 65 535, heads or kv_heads < 1, qld < heads 128, a row reading past cap or a smaller ws return RMU_ERR_ARG,
 * heads % kv_heads != 0 RMU_ERR_UNSUPPORTED. */
int rmu_debug_attention_decode_rows(const uint16_t* q_hi, const uint16_t* q_lo, int64_t qld, int B, const uint16_t* kv,
                                    int heads, int kv_heads, int cap, int P, const int32_t* pos_h, const int32_t* shift_h,
                                    float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* For tests: the batched prefill's attention (attention_causal_kernel over cached keys).  qkv planes [rows, (heads + 2
 * kv_heads) 128] hold only the own rows of B sequences (device cu [B + 1]); sequence b is P prefix rows then its own
 * rows, and every key comes from the cache kv [4][kv_heads, cap, 128]: key k at row k when k < P, else k +
 * shift[cu[b]] (device int32 per plane row).  -> ctx [rows, heads 128], each row equal to rmu_debug_attention_causal's
 * row on the full sequence.  max_own: the longest own part.  Null pointers, B outside 1 .. 65 535, heads, kv_heads
 * or max_own < 1, P < 0 or cap < P return RMU_ERR_ARG, heads % kv_heads != 0 RMU_ERR_UNSUPPORTED. */
int rmu_debug_attention_cached(const uint16_t* qkv_hi, const uint16_t* qkv_lo, const int32_t* cu, int B, int heads,
                               int kv_heads, const uint16_t* kv, int cap, int P, const int32_t* shift, int max_own,
                               uint16_t* ctx_hi, uint16_t* ctx_lo, void* stream);
/* For tests: decode attention, as rmu_decoder_generate runs it, of one query row q [heads 128] planes (pre-scaled by
 * log2(e) / sqrt(128)) against rows [0, n) of one layer's cache kv (fp16 planes K hi | K lo | V hi | V lo, each
 * [kv_heads, cap, 128]) -> ctx planes [heads 128]; query head h reads kv head h / (heads / kv_heads).  ws holds
 * heads * ceil(n / 64) * 130 floats.  Null pointers, heads or kv_heads < 1, n < 1, cap < n or a smaller ws return
 * RMU_ERR_ARG, heads % kv_heads != 0 RMU_ERR_UNSUPPORTED, before any CUDA call. */
int rmu_debug_attention_decode(const uint16_t* q_hi, const uint16_t* q_lo, const uint16_t* kv, int heads, int kv_heads,
                               int cap, int n, float* ws, int64_t ws_elems, uint16_t* ctx_hi, uint16_t* ctx_lo,
                               void* stream);
/* For tests: the KV-cache append of rmu_decoder_generate.  Copies the k and v heads of rows [0, T) of the planes hi / lo
 * [T, (heads + 2 kv_heads) 128] (q | k | v, as the q / k step leaves them) into rows pos0 .. pos0 + T - 1 of one layer's
 * cache kv (K hi | K lo | V hi | V lo, each [kv_heads, cap, 128]); nothing else of kv is written.  Null pointers, T,
 * heads or kv_heads < 1, pos0 < 0 or pos0 + T > cap return RMU_ERR_ARG, heads % kv_heads != 0 RMU_ERR_UNSUPPORTED,
 * before any CUDA call. */
/* The NF4 kernels one at a time (device pointers; fp16 planes as uint16).  quantize: hi [n] -> codes [n / 2], absmax
 * [n / 64]; dequantize: the reverse into hi [n]; gemv: one row x = x_hi + x_lo [K] against codes [N, K / 2] / absmax
 * [N, K / 64] with E1's epilogue `mode` at M = 1: 0 out_f32 [N] = acc + bias; 6 out_f32 = acc + bias + res_f32 (res_f32
 * may be out_f32); 7 SwiGLU on 128-row blocks of 64 gate | 64 up rows into out_hi / out_lo [N / 2], setting
 * *range_flag (nullable) when an output leaves the fp16 range.  Refused before any CUDA call: null pointers, n < 1,
 * a mode other than 0, 6, 7 (RMU_ERR_ARG); n or K not a multiple of 64, K > 49 152, N not a multiple of 128
 * (RMU_ERR_UNSUPPORTED).  nf4_conversion reads, for a converted handle, the most its conversion's allocations ever
 * exceeded the bytes held before it (<= 0) and their final difference, in bytes; RMU_ERR_ARG otherwise. */
int rmu_debug_nf4_quantize(const uint16_t* hi, int64_t n, uint8_t* codes, float* absmax, void* stream);
int rmu_debug_nf4_dequantize(const uint8_t* codes, const float* absmax, int64_t n, uint16_t* hi, void* stream);
int rmu_debug_nf4_gemv(int mode, const uint16_t* x_hi, const uint16_t* x_lo, const uint8_t* codes, const float* absmax,
                       int N, int K, const float* bias, const float* res_f32, float* out_f32, uint16_t* out_hi,
                       uint16_t* out_lo, int32_t* range_flag, void* stream);
int rmu_debug_nf4_conversion(const rmu_encoder* enc, int64_t* peak, int64_t* delta);
/* For tests: the batched decode's NF4 GEMV (rmu_decoder_generate_batch) on M rows x [M, K] (row pitch K) -> out_f32
 * [M, N] or out_hi / out_lo [M, N / 2]; res_f32 [M, N].  Row m's bits are rmu_debug_nf4_gemv's on row m alone.  The
 * arguments are refused as rmu_debug_nf4_gemv refuses them, and M outside 1..16 returns RMU_ERR_ARG. */
int rmu_debug_nf4_gemv_rows(int mode, int M, const uint16_t* x_hi, const uint16_t* x_lo, const uint8_t* codes,
                            const float* absmax, int N, int K, const float* bias, const float* res_f32, float* out_f32,
                            uint16_t* out_hi, uint16_t* out_lo, int32_t* range_flag, void* stream);
int rmu_debug_kv_append(const uint16_t* hi, const uint16_t* lo, int T, int heads, int kv_heads, int pos0, int cap,
                        uint16_t* kv, void* stream);
/* For tests: the sampler of rmu_decoder_generate on logits [V] (device fp32, overwritten with the processed values),
 * presence [ceil(V / 32)] (device, bit i of word i / 32 = id i is penalised; the chosen id's bit is set) and the
 * uniform u in [0, 1) -> *token (device int32).  The settings are refused as rmu_decoder_generate refuses them, and a
 * null pointer, V < 1 or u outside [0, 1) return RMU_ERR_ARG, before any CUDA call. */
int rmu_debug_sample(float* logits, int V, uint32_t* presence, const rmu_sampling* s, float u, int32_t* token,
                     void* stream);
/* For tests: the batched decode's sampler, one CTA per row r of logits [B, V] (device): the presence bits [.., ceil(V /
 * 32)] and Philox seed of sequence seq[r] (device int32 [B], device uint64 seeds), u = philox(seed, step) -> token[r].
 * Row r equals rmu_debug_sample on that row, those bits and that u.  Refused as rmu_debug_sample refuses, and a null
 * pointer, B < 1 or step < 0 return RMU_ERR_ARG. */
int rmu_debug_sample_rows(float* logits, int V, int B, uint32_t* presence, const int32_t* seq, const uint64_t* seeds,
                          int64_t step, const rmu_sampling* s, int32_t* token, void* stream);
/* For tests: a prompt-lookup verify pass's sampler.  Row j of logits [M, V] (device) samples with presence bits rows[j]
 * = presence | the bits of ids[1 .. j] (device ids [M]: the pending token, then the drafts; rows [M, ceil(V / 32)] is
 * written) and u = philox(seed, step0 + j) -> token[j]; presence is not written.  Refused as rmu_debug_sample refuses,
 * and a null pointer, M outside 1..16 or step0 < 0 return RMU_ERR_ARG. */
int rmu_debug_sample_verify_rows(float* logits, int V, int M, uint32_t* presence, const int32_t* ids, uint64_t seed,
                                 int64_t step0, const rmu_sampling* s, uint32_t* rows, int32_t* token, void* stream);
/* For tests and benchmarks: rmu_decoder_generate_lookup with the caller's drafts in place of the n-gram lookup: a pass
 * after n output tokens proposes drafts_h[n .. n + k) (host [max_new_tokens] ids in [0, vocab_size), k capped as
 * there).  Refused as rmu_decoder_generate_lookup refuses, and k < 0 or a draft id out of range (RMU_ERR_ARG). */
int rmu_debug_generate_drafts(rmu_encoder* enc, const int32_t* ids_h, int T, const rmu_sampling* s, uint64_t seed,
                              int max_new_tokens, const int32_t* drafts_h, int k, int32_t* out_h, int32_t* n_out,
                              float* logits_h, int32_t* n_passes, void* stream);
/* For tests: a decode session's sampler.  Row r of logits [B, V] (device) samples with the presence bits [.., ceil(V /
 * 32)], seed and Philox step of sequence seq[r] (device int32 [B], uint64 seeds and steps) and that sequence's settings
 * s_h[seq[r]] (host [n_seq]) -> token[r].  Row r equals rmu_debug_sample on that row, those bits, those settings and u =
 * philox(seed, step).  Refused as rmu_debug_sample refuses each s_h entry, and a null pointer, B < 1 or n_seq outside
 * 1..16 return RMU_ERR_ARG.  Synchronises `stream`. */
int rmu_debug_sample_session_rows(float* logits, int V, int B, uint32_t* presence, const int32_t* seq,
                                  const uint64_t* seeds, const uint64_t* steps, int n_seq, const rmu_sampling* s_h,
                                  int32_t* token, void* stream);
/* For tests (host only): a decode session's region placement.  Op i > 0 places ops[i] rows (first fit, growing past
 * the last used region when no gap fits) -> out[2 i] = the base; op i <= 0 frees the region at base -ops[i] -> out[2 i]
 * = 0, or -1 when no region starts there; out[2 i + 1] = the capacity after the op.  Null pointers or n < 0 return
 * RMU_ERR_ARG. */
int rmu_debug_kv_regions(const int32_t* ops, int n, int32_t* out);
int rmu_debug_split_planes(const float* src, int64_t n, uint16_t* hi, uint16_t* lo, void* stream);
int rmu_debug_join_planes(const uint16_t* hi, const uint16_t* lo, int64_t n, float* out, void* stream);
/* For tests: the BM25 select stage alone (bm25_select_kernel rounds, through the launcher rmu_bm25_search uses) on
 * caller-owned candidate lists: scores [Q, m] float64 and idx [Q, m] int32 document numbers (-1 = absent), each row
 * ascending in document number among its present entries, as stage 1 leaves them.  Scores hold no NaN and no -0.0 (the
 * scorer makes neither: every cell starts at +0.0, and +0.0 + -0.0 = +0.0).  Writes the top k of each row to out_scores
 * [Q, k] float64 and out_ids [Q, k] int64, score descending, equal scores by larger document number, -1 padded.
 * ws_scores and ws_idx are the ping-pong workspace, ws_elems elements each, at least 2 * Q * ceil(m / 4096) * k.  Null
 * pointers, Q < 1, m < 1 or a smaller workspace return RMU_ERR_ARG, and k outside 1..256 or Q > 65 535
 * RMU_ERR_UNSUPPORTED, before any CUDA call.  Allocates nothing. */
int rmu_debug_bm25_select(const double* scores, const int32_t* idx, int Q, int m, int k, double* ws_scores,
                          int32_t* ws_idx, int64_t ws_elems, double* out_scores, int64_t* out_ids, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RAGMEUP_B200_H */
