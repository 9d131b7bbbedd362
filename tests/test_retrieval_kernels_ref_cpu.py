"""CPU: pins the references of tests/test_retrieval_kernels_gpu.py (oracle/retrieval_kernels_ref.py) against the rank_bm25
and langchain restatements they stand in for."""
import numpy as np
import pytest

import cases
from oracle import flat_ref
from oracle import hybrid_ref as H
from oracle import retrieval_kernels_ref as R
from ragmeup_b200.bm25 import InvertedIndex


def _w(inv):
    return R.bm25_posting_weights(inv.post_ptr, inv.post_doc, inv.post_tf, inv.den, inv.idf, inv.k1 + 1)


@pytest.mark.parametrize("case", cases.BM25_CASES[:3], ids=lambda c: c["name"])
def test_vectorised_scorer_is_bit_identical_to_the_restatement(case):
    corpus, queries = cases.bm25_inputs(case)
    inv = InvertedIndex(corpus)
    bm = H.BM25Okapi(corpus)
    w = _w(inv)
    ids = [inv.term_ids(q) for q in queries]
    many = R.bm25_scores_many(inv.post_ptr, inv.post_doc, w, len(corpus), ids)
    for qi, q in enumerate(queries):
        want = bm.get_scores(q)
        got = R.bm25_scores(inv.post_ptr, inv.post_doc, w, len(corpus), ids[qi])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (case["name"], qi)
        assert np.array_equal(many[qi].view(np.uint64), want.view(np.uint64)), (case["name"], qi)
        ws, wd = H.bm25_topk(bm, q, case["k"])
        gs, gd = R.topk_stable(got, case["k"])
        assert np.array_equal(gd, wd) and np.array_equal(gs, ws)


def test_vectorised_scorer_with_negative_idf_repeats_and_other_parameters():
    # "a" is in every document: its idf is negative and floored at epsilon * average_idf, which is negative here
    corpus = [["a"] * (1 + i % 3) + ["b"] * (i % 2) for i in range(7)] + [["a", "c"]]
    q = [["a", "b", "a", "zzz", "c"], ["c"], ["b", "b"]]
    for params in (dict(), dict(k1=2.0, b=0.0), dict(k1=0.7, b=1.0, epsilon=0.5)):
        inv = InvertedIndex(corpus, **params)
        bm = H.BM25Okapi(corpus, **params)
        assert inv.average_idf < 0
        w = _w(inv)
        for qq in q:
            got = R.bm25_scores(inv.post_ptr, inv.post_doc, w, len(corpus), inv.term_ids(qq))
            assert np.array_equal(got.view(np.uint64), bm.get_scores(qq).view(np.uint64))
        assert (R.bm25_scores(inv.post_ptr, inv.post_doc, w, len(corpus), inv.term_ids(q[0])) < 0).any()


def test_select_reference_is_the_stable_argsort_order():
    rng = np.random.default_rng(3)
    for n, k, levels in ((50, 10, 4), (500, 256, 7), (3000, 37, 2), (9, 20, 3)):
        s = rng.integers(-levels, levels, n).astype(np.float64) * 0.375
        idx = np.arange(n, dtype=np.int32)
        gs, gi = R.select_ref(s[None], idx[None], k)
        ws, wi = R.topk_stable(s, k)
        kk = min(k, n)
        assert np.array_equal(gi[0, :kk], wi) and np.array_equal(gs[0, :kk], ws)
        assert (gi[0, kk:] == -1).all() and (gs[0, kk:] == 0.0).all()
    # absent entries are skipped, whatever score they carry
    s = np.array([[5.0, 9.0, 1.0, 9.0]])
    i = np.array([[2, -1, 7, 11]], dtype=np.int32)
    gs, gi = R.select_ref(s, i, 3)
    assert gi.tolist() == [[11, 2, 7]] and gs.tolist() == [[9.0, 5.0, 1.0]]


def test_mmr_witness_flips_between_double_and_float32_lambda():
    """the K6 case only means something if rounding lambda to float32 changes the answer"""
    q, E, lam = R.MMR_WITNESS_Q, R.MMR_WITNESS_E, R.MMR_WITNESS_LAMBDA
    assert flat_ref.mmr(q, E, lam, k=2) == [0, 1]
    assert flat_ref.mmr(q, E, float(np.float32(lam)), k=2) == [0, 2]
    assert R.mmr_replay(q, E, lam, 2, [0, 1]) == []
    assert R.mmr_replay(q, E, lam, 2, [0, 2])                # the float32 answer is more than tau from the best
    # the gap is about 1e6 tau at D = 3
    c = [R._cos(q, e) for e in E]
    sc = [lam * c[i] - (1 - lam) * R._cos(E[i], E[0]) for i in (1, 2)]
    assert 1e5 * R.mmr_tau(3) < sc[0] - sc[1] < 1e-9


@pytest.mark.parametrize("lam", [0.0, 0.3, 0.5, 1.0])
def test_mmr_replay_accepts_the_restatement_and_rejects_wrong_picks(lam):
    rng = np.random.default_rng(int(lam * 10) + 1)
    for n, d, k in ((20, 32, 10), (5, 3, 8), (64, 7, 64)):
        q = rng.standard_normal(d).astype(np.float32)
        E = rng.standard_normal((n, d)).astype(np.float32)
        want = flat_ref.mmr(q, E, lam, k)
        assert R.mmr_replay(q, E, lam, k, want + [-1] * (k - len(want))) == []
        bad = list(want)
        bad[1], bad[-1] = bad[-1], bad[1]
        assert R.mmr_replay(q, E, lam, k, bad + [-1] * (k - len(bad)))
        assert R.mmr_replay(q, E, lam, k, want + [-1] * (k - len(want)) + [0])       # wrong length
    # identical rows: the first one wins at every step
    E = np.ones((4, 3), np.float32)
    assert R.mmr_replay(np.ones(3, np.float32), E, lam, 4, [0, 1, 2, 3]) == []
    assert R.mmr_replay(np.ones(3, np.float32), E, lam, 4, [0, 2, 1, 3])
    assert R.mmr_replay(np.ones(3, np.float32), E, lam, 4, [3, 0, 1, 2])
