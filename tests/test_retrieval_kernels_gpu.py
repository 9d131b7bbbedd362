"""GPU: the retrieval-side kernels one at a time against float64 references, at the edges of their exact-semantics
promises (DESIGN.md §2).

* S1 ``bm25_score_kernel`` + ``bm25_select_kernel`` through ``BM25Index``: float64 scores and ids bit-identical to
  rank_bm25 (``oracle/retrieval_kernels_ref.py``, pinned against the restatement on the CPU) across three select rounds,
  term batches, CTA edges, negative scores and batches past 65 535 queries.
* S1 select rounds alone through ``rmu_debug_bm25_select`` against a lexsort.
* K6 ``mmr_kernel`` through ``mmr_select`` against a step-by-step fsum replay (the tolerance τ is derived in the
  oracle), K8 ``adjacent_cosine_kernel`` against numpy's cosine, K5 ``gather_rows_kernel`` bit for bit.
"""
import math

import numpy as np
import pytest

from oracle import chunker_ref, flat_ref
from oracle import hybrid_ref as H
from oracle import retrieval_kernels_ref as R

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


# ------------------------------------------------------------------ S1 through the product path
def _csr(n_docs, docs, terms, tfs):
    """(document, term, tf) triplets, one per (term, document) -> CSR by term, documents ascending, and lengths"""
    docs, terms, tfs = (np.asarray(a, dtype=np.int64) for a in (docs, terms, tfs))
    n_terms = int(terms.max()) + 1
    order = np.lexsort((docs, terms))
    post_ptr = np.zeros(n_terms + 1, dtype=np.int64)
    np.cumsum(np.bincount(terms, minlength=n_terms), out=post_ptr[1:])
    doc_len = np.bincount(docs, weights=tfs, minlength=n_docs).astype(np.int64)
    return post_ptr, docs[order].astype(np.int32), tfs[order].astype(np.int32), doc_len


def _first_seen(docs, terms):
    """renumber terms in first-seen order (documents ascending, then term order inside a document): rank_bm25 sums the
    idfs in that order, so any other numbering changes average_idf in the last bit"""
    terms = np.asarray(terms, dtype=np.int64)
    order = np.lexsort((np.arange(len(docs)), docs))
    _, first = np.unique(terms[order], return_index=True)
    seen = terms[order][np.sort(first)]
    remap = np.empty(int(terms.max()) + 1, dtype=np.int64)
    remap[seen] = np.arange(len(seen))
    return remap[terms]


def _index(n_docs, docs, terms, tfs, **params):
    from ragmeup_b200.bm25 import BM25Index
    terms = _first_seen(docs, terms)
    post_ptr, post_doc, post_tf, doc_len = _csr(n_docs, docs, terms, tfs)
    idx = BM25Index.from_arrays(post_ptr, post_doc, post_tf, doc_len, **params)
    idx.w = R.bm25_posting_weights(idx.post_ptr, idx.post_doc, idx.post_tf, idx.den, idx.idf, idx.k1 + 1)
    return idx


def _token_lists(idx):
    """the corpus as rank_bm25 sees it: document d holds [str(t)] * tf for its terms, in first-seen order"""
    out = [[] for _ in range(idx.corpus_size)]
    term = np.repeat(np.arange(len(idx.post_ptr) - 1), np.diff(idx.post_ptr))
    for t, d, f in sorted(zip(term.tolist(), idx.post_doc.tolist(), idx.post_tf.tolist()), key=lambda e: (e[1], e[0])):
        out[d] += [str(t)] * f
    return out


def _check_search(idx, queries, k, restatement=False):
    """search -> bit-identical to the vectorised rank_bm25 scorer's stable top k (and to the restatement itself)"""
    s, d = idx.search(queries, k)
    bm = H.BM25Okapi(_token_lists(idx), idx.k1, idx.b, idx.epsilon) if restatement else None
    for qi, q in enumerate(queries):
        full = R.bm25_scores(idx.post_ptr, idx.post_doc, idx.w, idx.corpus_size, idx.term_ids(q))
        ws, wd = R.topk_stable(full, k)
        assert np.array_equal(d[qi], wd), (qi, d[qi][:8], wd[:8])
        assert np.array_equal(_bits(s[qi]), _bits(ws)), qi
        if bm is not None:
            assert np.array_equal(_bits(bm.get_scores(q)), _bits(full))
    return s, d


def test_bm25_million_document_tie_takes_three_select_rounds(cuda):
    from ragmeup_b200 import _lib
    n, k = 1_050_000, 256                # 257 CTAs -> 65 792 -> 4 352 -> 512 -> 256 candidates
    idx = _index(n, np.arange(n), np.zeros(n, np.int64), np.ones(n, np.int64))
    l0 = _lib.launch_count()
    s, d = idx.search([["0"]], k)
    assert _lib.launch_count() - l0 == 4                 # stage 1 + three select rounds
    assert d[0].tolist() == list(range(n - 1, n - 1 - k, -1))
    assert (_bits(s[0]) == _bits(idx.w[0])).all() and s[0, 0] < 0          # one term in every document: idf floored
    _check_search(idx, [["0"]], k)


def test_bm25_top_k_with_positive_zero_and_negative_scores(cuda):
    # term 0 in every document and term 1 in all but two pull average_idf below 0, so the epsilon floor is negative
    n = 40
    docs = [*range(n), *range(n - 2), 3, 17, 30]
    terms = [0] * n + [1] * (n - 2) + [2, 2, 2]
    tfs = [1 + d % 3 for d in range(n)] + [1 + d % 2 for d in range(n - 2)] + [1, 4, 2]
    idx = _index(n, docs, terms, tfs)
    assert idx.average_idf < 0
    s, _ = _check_search(idx, [["2", "1"], ["1", "2", "2"], ["2"]], n, restatement=True)
    assert (s[0] > 0).any() and (s[0] < 0).any() and (_bits(s[0]) == 0).sum() == 2       # +0.0, not -0.0
    assert (s[2] > 0).sum() == 3 and (_bits(s[2]) == 0).sum() == n - 3


def test_bm25_queries_across_the_term_batch(cuda):
    rng = np.random.default_rng(5)
    n, vocab = 9000, 700                                 # three CTAs
    lens = rng.integers(1, 12, n)
    docs = np.repeat(np.arange(n), lens)
    terms = np.concatenate([rng.choice(vocab, size=m, replace=False) for m in lens])
    idx = _index(n, docs, terms, rng.integers(1, 6, len(docs)))
    live = [str(t) for t in range(len(idx.idf)) if idx.idf[t] != 0.0]
    queries = []
    for m in (255, 256, 257, 512, 513):
        q = [str(t) for t in rng.choice(live, size=m - 40)] + [str(t) for t in rng.choice(live[:20], size=40)]
        q.insert(m // 2, "not-a-term")
        assert len(idx.term_ids(q)) == m
        queries.append(q)
    _check_search(idx, queries, 256)
    _check_search(idx, queries, 7)


@pytest.mark.parametrize("n", [4095, 4096, 4097, 3 * 4096 - 1, 3 * 4096, 3 * 4096 + 1])
def test_bm25_corpus_sizes_at_the_cta_edge(cuda, n):
    rng = np.random.default_rng(n)
    lens = rng.integers(1, 4, n)
    docs = np.repeat(np.arange(n), lens)
    terms = np.concatenate([rng.choice(12, size=m, replace=False) for m in lens])   # few terms: many ties
    idx = _index(n, docs, terms, rng.integers(1, 3, len(docs)))
    queries = [["0"], ["1", "5"], ["2", "2", "7", "11"], [str(t) for t in range(12)]]
    for k in (1, 255, 256):
        _check_search(idx, queries, k)


def test_bm25_large_tf_empty_documents_and_extreme_parameters(cuda):
    # tf up to 1e6 and empty documents, default and b = 0 (restatement checked); b = 1 without empty documents
    docs = [0, 0, 1, 2, 2, 4, 5, 5, 7]
    terms = [0, 1, 0, 1, 2, 0, 2, 1, 1]
    tfs = [1_000_000, 1, 999_999, 3, 1, 1, 500_000, 2, 1]
    q = [["0"], ["1", "0", "2"], ["2", "1", "1"]]
    for params in (dict(), dict(b=0.0), dict(k1=2.0, b=0.0)):
        _check_search(_index(9, docs, terms, tfs, **params), q, 9, restatement=True)     # documents 3, 6, 8 are empty
    full = [0, 0, 1, 2, 2, 3, 4, 4, 5, 6, 7, 8]
    fterms = [0, 1, 0, 1, 2, 1, 2, 1, 0, 2, 1, 0]
    ftfs = [1_000_000, 1, 999_999, 3, 1, 7, 500_000, 2, 1, 1, 1, 40]
    _check_search(_index(9, full, fterms, ftfs, b=1.0), q, 9, restatement=True)
    # k1 = 0: every posting weighs exactly idf.  rank_bm25 divides 0 by 0 for a document without the term and scores
    # it NaN; the kernel and the vectorised reference add nothing, so only the posting-wise reference applies here
    idx = _index(9, full, fterms, ftfs, k1=0.0, b=0.75)
    assert (idx.w == idx.idf[np.repeat(np.arange(3), np.diff(idx.post_ptr))]).all()
    _check_search(idx, q, 9)


def test_bm25_batches_past_the_grid_limit(cuda):
    """the query index is gridDim.y: 65 536 and more queries run in chunks of 65 535"""
    rng = np.random.default_rng(11)
    n, vocab, Q, k = 300, 40, 65_537, 5
    lens = rng.integers(1, 8, n)
    docs = np.repeat(np.arange(n), lens)
    terms = np.concatenate([rng.choice(vocab, size=m, replace=False) for m in lens])
    idx = _index(n, docs, terms, rng.integers(1, 4, len(docs)))
    qlen = rng.integers(1, 5, Q)
    qt = rng.integers(0, vocab, int(qlen.sum()))
    ids = np.split(qt, np.cumsum(qlen)[:-1])
    queries = [[str(t) for t in row] for row in ids]
    full = R.bm25_scores_many(idx.post_ptr, idx.post_doc, idx.w, n, [idx.term_ids(q) for q in queries])
    top = np.argsort(full, axis=1, kind="stable")[:, ::-1][:, :k]
    want_s = np.take_along_axis(full, top, axis=1)
    for nq in (65_535, 65_536, Q):
        s, d = idx.search(queries[:nq], k)
        bad = np.flatnonzero((d != top[:nq]).any(1) | (_bits(s) != _bits(want_s[:nq])).any(1))
        assert bad.size == 0, (nq, bad[:10])


# ------------------------------------------------------------------ S1 select alone
def _select(scores, idx, k):
    import torch
    from ragmeup_b200 import _lib
    Q, m = scores.shape
    half = Q * ((m + 4095) // 4096) * k
    dev = torch.device("cuda")
    s = torch.from_numpy(np.ascontiguousarray(scores, np.float64)).to(dev)
    i = torch.from_numpy(np.ascontiguousarray(idx, np.int32)).to(dev)
    ws_s = torch.full((2 * half,), float("nan"), dtype=torch.float64, device=dev)
    ws_i = torch.full((2 * half,), -7, dtype=torch.int32, device=dev)
    out_s = torch.full((Q, k), float("nan"), dtype=torch.float64, device=dev)
    out_i = torch.full((Q, k), -7, dtype=torch.int64, device=dev)
    l0 = _lib.launch_count()
    _lib.check(_lib.lib().rmu_debug_bm25_select(s.data_ptr(), i.data_ptr(), Q, m, k, ws_s.data_ptr(), ws_i.data_ptr(),
                                                2 * half, out_s.data_ptr(), out_i.data_ptr(), _lib.stream_ptr()),
               "rmu_debug_bm25_select")
    torch.cuda.synchronize()
    return out_s.cpu().numpy(), out_i.cpu().numpy(), _lib.launch_count() - l0


def _rounds(m, k):
    r = 1
    while m > 4096:
        m, r = (m + 4095) // 4096 * k, r + 1
    return r


def _check_select(scores, idx, k):
    gs, gi, launches = _select(scores, idx, k)
    ws, wi = R.select_ref(scores, idx, k)
    for r in range(scores.shape[0]):
        assert np.array_equal(gi[r], wi[r]), (r, gi[r][:8], wi[r][:8])
        assert np.array_equal(_bits(gs[r]), _bits(ws[r])), r
    assert launches == _rounds(scores.shape[1], k)


def _ascending_ids(rng, Q, m, absent=0.0):
    """document numbers strictly ascending along each row (gaps 1..999, below 2^31), a share of them absent (-1)"""
    ids = np.cumsum(rng.integers(1, 1000, (Q, m)), axis=1).astype(np.int32)
    if absent:
        ids[rng.random((Q, m)) < absent] = -1
    return ids


def test_select_keys_equal_in_their_top_seven_bytes(cuda):
    rng = np.random.default_rng(1)
    m, k = 9000, 100
    for base in (1.2345, -1.2345, 7e-300, -3e200):
        bits = np.full(m, np.float64(base).view(np.uint64)) ^ rng.integers(0, 256, m).astype(np.uint64)
        _check_select(bits.view(np.float64)[None], _ascending_ids(rng, 1, m), k)


@pytest.mark.parametrize("byte", range(8))
def test_select_exactly_k_keys_at_a_radix_bucket_boundary(cuda, byte):
    """k keys of x and the rest of y < x, x and y differing in one byte: the pass on that byte finds exactly k keys in
    the top bucket, the case `hist[b] >= remaining` has to take"""
    rng = np.random.default_rng(byte)
    k = 64
    y = np.float64(3.5).view(np.uint64) & ~np.uint64(0xFF << (8 * (7 - byte)) if byte else 0x7F << 56)
    x = y | np.uint64(0x01 << (8 * (7 - byte)))
    for m, where in ((4096, "spread"), (20000, "spread"), (20000, "one cta")):
        s = np.full(m, y).view(np.float64)
        pos = rng.choice(m, k, replace=False) if where == "spread" else np.arange(5000, 5000 + k)
        s[pos] = np.array(x).view(np.float64)
        assert (s > s.min()).sum() == k
        _check_select(s[None].copy(), _ascending_ids(rng, 1, m), k)


def test_select_absent_entries_and_short_rows(cuda):
    rng = np.random.default_rng(2)
    m, k = 12_000, 200
    s = rng.integers(-30, 30, (6, m)) * 0.25
    ids = _ascending_ids(rng, 6, m, absent=0.3)
    s[ids < 0] = 1e300                                   # an absent entry must never be taken, whatever its score
    ids[1, :] = -1                                       # nothing valid
    for row, n_valid in ((2, 7), (3, k), (4, k + 1), (5, k - 1)):
        live = np.sort(rng.choice(m, n_valid, replace=False))
        ids[row, :] = -1
        ids[row, live] = np.sort(rng.choice(1 << 30, n_valid, replace=False))
    _check_select(s, ids, k)
    _check_select(s[:, :4096], ids[:, :4096], 256)


@pytest.mark.parametrize("r", [1, 2, 17, 300])
def test_select_lengths_around_cta_multiples(cuda, r):
    rng = np.random.default_rng(r)
    for m in (4096 * r - 1, 4096 * r + 1):
        Q = 2 if r < 300 else 1
        s = rng.integers(-50, 50, (Q, m)) * 0.125                       # ties everywhere, negative scores included
        ids = _ascending_ids(rng, Q, m)
        for k in ((1, 256) if r == 300 else (1, 129, 256)):
            _check_select(s, ids, k)


def test_select_ties_across_cta_boundaries_in_every_round(cuda):
    rng = np.random.default_rng(4)
    m = 1_100_000                                        # 269 -> 17 -> 2 -> 1 CTAs at k = 256
    ids = _ascending_ids(rng, 1, m)
    _check_select(np.full((1, m), -2.75), ids, 256)
    # two levels: the best 300 (more than k) straddle the boundaries of every round's CTAs
    s = np.full((1, m), -3.0)
    s[0, rng.choice(m, 300, replace=False)] = -1.5
    _check_select(s, ids, 256)
    _check_select(s, ids, 255)


# ------------------------------------------------------------------ K6
def _mmr(q, cand, n_cand, k, lam):
    import torch
    from ragmeup_b200.index import mmr_select
    nc = None if n_cand is None else torch.as_tensor(np.asarray(n_cand, np.int32), device="cuda")
    out = mmr_select(torch.as_tensor(q, device="cuda"), torch.as_tensor(cand, device="cuda"), nc, k, lam)
    return out.cpu().numpy()


def _check_mmr(q, cand, n_cand, k, lam, got):
    for b in range(len(q)):
        n = cand.shape[1] if n_cand is None else min(int(n_cand[b]), cand.shape[1])
        want = flat_ref.mmr(q[b], cand[b, :n], lam, k)
        if got[b].tolist() == want + [-1] * (k - len(want)):
            continue                                     # numpy's own pick is within tau of the best at every step
        errs = R.mmr_replay(q[b], cand[b, :n], lam, k, got[b].tolist())
        assert not errs, (b, n, k, lam, errs)


@pytest.mark.parametrize("fetch_k", [1, 2, 20, 63, 64])
def test_mmr_shapes_and_lambdas(cuda, fetch_k):
    rng = np.random.default_rng(fetch_k)
    lams = [0.0, 0.25, 0.3, 0.5, 0.7, 1.0]
    for j, D in enumerate((1, 3, 31, 32, 33, 384, 1536)):
        n_cand = sorted({0, 1, max(fetch_k - 1, 0), fetch_k, fetch_k + 5})
        nq = len(n_cand)
        q = rng.standard_normal((nq, D)).astype(np.float32)
        cand = rng.standard_normal((nq, fetch_k, D)).astype(np.float32)
        # near-duplicates make the redundancy term matter
        cand[:, 1::3] = cand[:, 0:1] + 0.1 * cand[:, 1::3]
        for lam in (lams[j % 6], lams[(j + 3) % 6]):
            for k in (min(4, fetch_k), fetch_k + 2):     # k > n pads with -1
                got = _mmr(q, cand, n_cand, k, lam)
                _check_mmr(q, cand, n_cand, k, lam, got)
                assert (got[0] == -1).all()               # n_cand = 0


def test_mmr_degenerate_candidates(cuda):
    rng = np.random.default_rng(9)
    D, fk, k = 33, 20, 24
    v = rng.standard_normal(D).astype(np.float32)
    same = np.broadcast_to(v, (fk, D))
    anti = np.where(np.arange(fk)[:, None] % 2 == 0, v, -v).astype(np.float32)
    mixed = rng.standard_normal((fk, D)).astype(np.float32)
    mixed[[4, 9, 15]] = mixed[2]                         # exact duplicates of candidate 2
    cand = np.stack([same, np.zeros((fk, D), np.float32), anti, mixed, same]).astype(np.float32)
    q = np.stack([v, v, v, rng.standard_normal(D), np.zeros(D)]).astype(np.float32)    # last: zero query
    for lam in (0.0, 0.3, 0.5, 1.0):
        got = _mmr(q, cand, None, k, lam)
        _check_mmr(q, cand, None, k, lam, got)
        pad = [-1] * (k - fk)
        assert got[0].tolist() == list(range(fk)) + pad              # identical candidates: 0, 1, 2, ...
        assert got[1].tolist() == list(range(fk)) + pad              # zero candidates
        assert got[4].tolist() == list(range(fk)) + pad              # identical candidates, zero query
        assert got[2, 0] == 0 and (lam >= 0.5 or got[2, 1] == 1)     # below 0.5 the anti-parallel row comes second


def test_mmr_many_queries_and_the_refusals(cuda):
    from ragmeup_b200 import _lib
    rng = np.random.default_rng(12)
    nq, fk, D = 4097, 20, 32
    q = rng.standard_normal((nq, D)).astype(np.float32)
    cand = rng.standard_normal((nq, fk, D)).astype(np.float32)
    n_cand = rng.integers(0, fk + 3, nq)
    got = _mmr(q, cand, n_cand, 10, 0.7)
    _check_mmr(q, cand, n_cand, 10, 0.7, got)
    with pytest.raises(_lib.RmuError):
        _mmr(q[:2], rng.standard_normal((2, 65, D)).astype(np.float32), None, 4, 0.5)      # fetch_k > 64


def test_mmr_lambda_is_a_double(cuda):
    """lambda rounded to float32 flips this near-tie (tests/test_retrieval_kernels_ref_cpu.py pins the flip)"""
    import torch
    from ragmeup_b200.vectorstore import Milvus
    q, E, lam = R.MMR_WITNESS_Q, R.MMR_WITNESS_E, R.MMR_WITNESS_LAMBDA
    assert _mmr(q[None], E[None], None, 2, lam).tolist() == [[0, 1]]
    assert _mmr(q[None], E[None], None, 2, float(np.float32(lam))).tolist() == [[0, 2]]

    class Emb:
        def embed_documents(self, texts):
            return [[0.0, 0.0, 0.0] for _ in texts]

        def embed_query(self, text):
            return [0.0, 0.0, 0.0]

    db = Milvus(Emb(), collection_name="witness")
    db.add_embeddings(E, ["a", "b", "c"])
    rows = db.mmr_tensor(torch.as_tensor(q[None], device="cuda"), k=2, fetch_k=3, lambda_mult=lam)
    assert rows.cpu().tolist() == flat_ref.mmr_search(q[None], E, 2, "l2", fetch_k=3, lambda_mult=lam) == [[0, 1]]


# ------------------------------------------------------------------ K8
def _adjacent_ref(x):
    """1 - cosine_similarity of consecutive rows, float64, NaN and +-inf similarities -> 0 (vectorised)"""
    X = np.asarray(x, dtype=np.float64)
    nrm = np.linalg.norm(X, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        sim = np.einsum("ij,ij->i", X[:-1], X[1:]) / (nrm[:-1] * nrm[1:])
    sim[~np.isfinite(sim)] = 0.0
    return 1.0 - sim


@pytest.mark.parametrize("D", [1, 31, 32, 33, 4096])
def test_adjacent_distance_shapes_zero_rows_and_magnitudes(cuda, D):
    import torch
    from ragmeup_b200.chunker import adjacent_cosine_distance
    rng = np.random.default_rng(D)
    n = 40
    x = rng.standard_normal((n, D)) * 10.0 ** rng.uniform(-30, 30, (n, 1))      # magnitudes 1e-30 .. 1e30
    zero = [0, 17, 25, 26, n - 1]                        # first, middle, two adjacent, last
    x[zero] = 0.0
    x = x.astype(np.float32)
    got = adjacent_cosine_distance(torch.as_tensor(x, device="cuda"))
    touches = sorted({p for z in zero for p in (z - 1, z) if 0 <= p < n - 1})
    assert (got[touches] == 1.0).all(), got[touches]
    with np.errstate(divide="ignore", invalid="ignore"):
        small = np.asarray(chunker_ref.distances_from_embeddings(x.tolist()))
    assert np.array_equal(_adjacent_ref(x)[touches], small[touches])
    assert np.abs(_adjacent_ref(x) - small).max() < 1e-12 and np.abs(got - small).max() < 1e-12


def test_adjacent_distance_hundred_thousand_pairs(cuda):
    import torch
    from ragmeup_b200.chunker import adjacent_cosine_distance
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(100_001, 96, device="cuda", generator=g) * torch.rand(100_001, 1, device="cuda", generator=g)
    x[::1000] = 0.0
    got = adjacent_cosine_distance(x)
    want = _adjacent_ref(x.cpu().numpy())
    assert got.shape == (100_000,) and np.abs(got - want).max() < 1e-12
    assert (got[::1000] == 1.0).all() and (got[999::1000] == 1.0).all()


# ------------------------------------------------------------------ K5
def test_gather_rows_out_of_range_are_zero(cuda):
    import torch
    from ragmeup_b200.index import FlatIndex
    rng = np.random.default_rng(8)
    n, D = 1000, 33
    x = rng.standard_normal((n, D)).astype(np.float32)
    x[5] = np.float32(1e-42)                              # subnormals copy as they are
    index = FlatIndex(D, "l2")
    index.add(x)
    rows = np.array([3, -1, 5, n, n + 5, 2 ** 40, n - 1, 0, -(2 ** 40), 999, 5], dtype=np.int64)
    got = index.gather(torch.as_tensor(rows, device="cuda")).cpu().numpy()
    valid = (rows >= 0) & (rows < n)
    assert np.array_equal(got[valid].view(np.uint32), x[rows[valid]].view(np.uint32))
    assert np.array_equal(got[~valid].view(np.uint32), np.zeros(((~valid).sum(), D), np.uint32))
    assert math.isclose(float(got[2, 0]), 1e-42, rel_tol=1e-2)
