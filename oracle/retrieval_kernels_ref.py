"""References for the retrieval-side kernels tested one at a time: S1 (BM25 scoring and select), K6 (MMR).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``); pinned on the CPU by ``tests/test_retrieval_kernels_ref_cpu.py``.

* ``bm25_posting_weights`` / ``bm25_scores`` / ``bm25_scores_many``: rank_bm25's ``get_scores`` over CSR postings,
  vectorised.  rank_bm25 evaluates ``idf * (tf * (k1 + 1) / (tf + den))`` for every document and adds it to the score,
  term by term in query order; a document without the term adds ``idf * 0 / den = +-0.0``, which leaves any score
  unchanged (scores start at +0.0 and ``+0.0 + -0.0 = +0.0``).  Adding only the postings therefore gives the same
  float64 bits, as long as ``den > 0`` (with ``k1 = 0``, or ``b = 1`` on an empty document, rank_bm25 divides 0 by 0 and
  scores NaN; these functions, like the kernel, add nothing).  numpy's elementwise operations do not contract to FMA.
* ``topk_stable``: ``np.argsort(scores, kind="stable")[::-1][:k]``, the order ``hybrid_ref.bm25_topk`` pins.
* ``select_ref``: the select stage on candidate lists: score descending, equal scores by larger document number.
* ``mmr_replay``: replays a greedy MMR selection step by step with ``math.fsum`` dots and norms (see ``mmr_tau``).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np

U64 = 2.0 ** -53          # float64 unit roundoff

# A near-tie that float32(0.3) flips (vectors are float32, exact as written): langchain's MMR with the Python double
# 0.3 picks [0, 1] (score gap +5.4e-10); with lambda rounded to float32 it picks [0, 2] (gap -3.3e-10).
MMR_WITNESS_Q = np.array([1.0, 0.0, 0.0], dtype=np.float32)
MMR_WITNESS_E = np.array([[1.0, 0.05000000074505806, 0.0],
                          [1.8016349077224731, 1.3151037693023682, 0.3573804199695587],
                          [1.0540894269943237, -0.004454133100807667, 0.6564749479293823]], dtype=np.float32)
MMR_WITNESS_LAMBDA = 0.3


# ------------------------------------------------------------------ S1
def bm25_posting_weights(post_ptr, post_doc, post_tf, den, idf, k1p1) -> np.ndarray:
    """float64 [nnz]: idf[t] * (tf * k1p1 / (tf + den[doc])) for every posting, rank_bm25's operation order"""
    term = np.repeat(np.arange(len(post_ptr) - 1), np.diff(post_ptr))
    tf = np.asarray(post_tf, dtype=np.float64)
    return np.asarray(idf, dtype=np.float64)[term] * (tf * k1p1 / (tf + np.asarray(den, dtype=np.float64)[post_doc]))


def bm25_scores(post_ptr, post_doc, w, n_docs: int, q_terms: Sequence[int]) -> np.ndarray:
    """float64 [n_docs]: one query's scores, terms added in query order (repeats kept)"""
    score = np.zeros(n_docs)
    for t in q_terms:
        p0, p1 = int(post_ptr[t]), int(post_ptr[t + 1])
        score[post_doc[p0:p1]] += w[p0:p1]          # one posting per (term, document): no repeated index
    return score


def bm25_scores_many(post_ptr, post_doc, w, n_docs: int, queries: Sequence[Sequence[int]]) -> np.ndarray:
    """float64 [Q, n_docs] for a small corpus: term j of every query is added in one step (per row, rank_bm25's order)"""
    n_terms = len(post_ptr) - 1
    dense = np.zeros((n_terms, n_docs))
    dense[np.repeat(np.arange(n_terms), np.diff(post_ptr)), post_doc] = w
    out = np.zeros((len(queries), n_docs))
    lens = np.asarray([len(q) for q in queries])
    for j in range(int(lens.max(initial=0))):
        rows = np.flatnonzero(lens > j)
        out[rows] += dense[[queries[r][j] for r in rows]]
    return out


def topk_stable(scores: np.ndarray, k: int):
    """(scores, ids int64) of the k best, ``argsort(kind="stable")[::-1]`` order: equal scores -> larger index first"""
    top = np.argsort(scores, kind="stable")[::-1][:k]
    return scores[top], top.astype(np.int64)


def select_ref(scores: np.ndarray, idx: np.ndarray, k: int):
    """select stage on candidate lists [Q, m] (idx -1 = absent) -> (scores [Q, k], ids int64 [Q, k]): score
    descending, equal scores by larger document number; missing entries are (0.0, -1) as the kernel writes them"""
    Q = scores.shape[0]
    out_s = np.zeros((Q, k))
    out_i = np.full((Q, k), -1, dtype=np.int64)
    for r in range(Q):
        live = np.flatnonzero(idx[r] >= 0)
        s, d = scores[r, live], idx[r, live].astype(np.int64)
        order = np.lexsort((-d, -s))[:k]                # last key is primary
        out_s[r, :len(order)] = s[order]
        out_i[r, :len(order)] = d[order]
    return out_s, out_i


# ------------------------------------------------------------------ K6
def mmr_tau(dim: int) -> float:
    """How far the kernel's MMR score may sit from the replay's.

    The kernel forms every dot product of float32 inputs in float64: the products are exact (24 x 24 bits), and any
    order of D - 1 additions is within (D - 1)·u·Σ|a b| ≤ (D - 1)·u·‖a‖‖b‖ (Cauchy–Schwarz), u = 2⁻⁵³.  So the dot is
    within (D - 1)·u of ‖a‖‖b‖, each norm within ((D - 1)/2 + 1)·u relative (sum, then sqrt), and the product and the
    quotient add u each: |Δcos| ≤ (2D + 2)·u.  The replay's cosines (fsum, sqrt, product, quotient) are within 4u of
    exact.  The MMR score λ·a − (1 − λ)·b with λ in [0, 1] moves by at most max|Δcos| plus 3u of its own rounding on
    each side: τ = (2D + 2 + 4 + 6)·u, rounded up to (2D + 16)·u."""
    return (2 * dim + 16) * U64


def _norm(a) -> float:
    a = np.asarray(a, dtype=np.float64)
    return math.sqrt(math.fsum(a * a))


def _cos(a, b, na: Optional[float] = None, nb: Optional[float] = None) -> float:
    """cosine_similarity's value (NaN and +-inf -> 0) from correctly rounded sums; na / nb: norms already computed"""
    den = (_norm(a) if na is None else na) * (_norm(b) if nb is None else nb)
    if den == 0.0:
        return 0.0
    c = math.fsum(np.asarray(a, dtype=np.float64) * np.asarray(b, dtype=np.float64)) / den
    return c if math.isfinite(c) else 0.0


def mmr_replay(q, E, lambda_mult: float, k: int, picks: Sequence[int], tau: Optional[float] = None) -> List[str]:
    """Check a greedy MMR selection (langchain ``maximal_marginal_relevance``) step by step; returns the failures.

    At every step the pick must be an unchosen candidate whose score is within τ of the best score, and no unchosen
    candidate before it may hold an identical row (equal rows give bit-equal scores in the kernel and in numpy, so
    the first maximum wins there).  Within τ the replay cannot tell which candidate numpy would pick, so it follows
    the pick.  After min(k, n) picks the rest must be -1."""
    E = np.asarray(E, dtype=np.float32)
    n = E.shape[0]
    tau = mmr_tau(E.shape[1] if E.ndim == 2 else 1) if tau is None else tau
    kk = min(k, n)
    picks = [int(p) for p in picks]
    errs = []
    if len(picks) != k or any(p != -1 for p in picks[kk:]):
        errs.append(f"expected {kk} picks then -1 padding to {k}, got {picks}")
    norms = [_norm(E[i]) for i in range(n)]
    qn = _norm(q)
    cos_q = [_cos(q, E[i], qn, norms[i]) for i in range(n)]
    best = [-math.inf] * n
    chosen: List[int] = []
    for step in range(kk):
        p = picks[step] if step < len(picks) else -1
        live = [i for i in range(n) if i not in chosen]
        if step == 0:
            sc = {i: cos_q[i] for i in live}
        else:
            sc = {i: lambda_mult * cos_q[i] - (1 - lambda_mult) * best[i] for i in live}
        top = max(sc.values())
        if p not in sc:
            errs.append(f"step {step}: pick {p} is not an unchosen candidate")
            break
        if sc[p] < top - tau:
            errs.append(f"step {step}: pick {p} scores {sc[p]!r}, best {top!r} (tau {tau:.3g})")
        dup = [i for i in live if i < p and np.array_equal(E[i], E[p])]
        if dup:
            errs.append(f"step {step}: pick {p} has an identical earlier candidate {dup[0]}")
        chosen.append(p)
        for i in range(n):
            best[i] = max(best[i], _cos(E[i], E[p], norms[i], norms[p]))
    return errs
