"""GPU: the FlashrankRerank drop-in on the sm_90a encoder against oracle/flashrank_ref.py over bert_ref's fp32
forward, at the three FlashRank BERT shapes, and wired as RAGMeUp wires its default reranker
(server/RAGHelper.py:476-490; rerank provenance, server/provenance.py:100-108)."""
import threading
from dataclasses import asdict

import numpy as np
import pytest
from tokenizers import Tokenizer

from oracle import bert_ref, flat_ref
from oracle import flashrank_ref as FR
from oracle import hybrid_ref as H
from oracle import provenance_ref as P
from ragmeup_b200.documents import Document
from ragmeup_b200.tokenizer import synthetic_sentences, synthetic_vocab

pytestmark = pytest.mark.gpu

SHAPES = ["ms-marco-MultiBERT-L-12", "ms-marco-TinyBERT-L-2-v2", "ms-marco-MiniLM-L-12-v2"]
PADS = [" ", "\t", "\n ", "  \r\n", ""]


@pytest.fixture(scope="module")
def model(cuda):
    """name -> (Ranker, oracle cfg, weights, private tokenizer copy for the oracle), built once per name; the
    encoders are released when the module ends, not at interpreter exit"""
    from ragmeup_b200.flashrank import Ranker
    from ragmeup_b200.weights import resolve_flashrank
    cache = {}

    def get(name):
        if name not in cache:
            r = Ranker(name)
            cfg, w, max_len, _ = resolve_flashrank(name)
            assert max_len == r.max_length == 512
            cache[name] = (r, bert_ref.BertCfg(**asdict(cfg)), w, Tokenizer.from_str(r.tokenizer.to_str()))
        return cache[name]
    yield get
    cache.clear()


def _pad(texts, seed):
    rng = np.random.default_rng(seed)
    return [PADS[int(rng.integers(len(PADS)))] + t + PADS[int(rng.integers(len(PADS)))] for t in texts]


def _call_shape(vocab, seed):
    """RAGMeUp's rerank call: a ~16-token query against 14 documents of ~130 tokens, plus one truncated at 512"""
    q = _pad(synthetic_sentences(vocab, 1, 14, 18, seed=seed), seed + 1)[0]
    docs = synthetic_sentences(vocab, 14, 110, 150, seed=seed + 2) + synthetic_sentences(vocab, 1, 600, 700, seed=seed + 3)
    return q, _pad(docs, seed + 4)


def _score_bound(cfg):
    """|d score| per 1e-3 of logit error: sigmoid' <= 1/4; d softmax_1 <= (|d l_0| + ... ) / 4 over the labels"""
    return 0.25e-3 * (1 if cfg.num_labels == 1 else cfg.num_labels)


def _check_order(got_ids, ref_scores, bound):
    """every pair the oracle separates by more than twice the propagated bound comes out in the oracle's order"""
    pos = {i: k for k, i in enumerate(got_ids)}
    for i in range(len(ref_scores)):
        for j in range(len(ref_scores)):
            if ref_scores[i] - ref_scores[j] > 2 * bound:
                assert pos[i] < pos[j], (i, j, ref_scores[i], ref_scores[j])


@pytest.mark.parametrize("scale", [1.0, 4.0])
@pytest.mark.parametrize("preset", SHAPES)
def test_logits_order_and_scores_match_the_oracle(model, preset, scale):
    from ragmeup_b200.flashrank import FlashrankRerank
    name = f"synthetic:{preset}:3:{scale}"
    r, ocfg, w, otok = model(name)
    vocab = synthetic_vocab(ocfg.vocab_size)
    for seed in (10, 20):
        q, texts = _call_shape(vocab, seed)
        ids, _, cu = r._pairs([q] * len(texts), texts)
        assert int(np.max(np.diff(cu))) == 512
        if ocfg.vocab_size > 30522:
            assert int(ids.max()) > 30521                          # the multilingual rows of the embedding table
        lib = r.logits(q, texts)
        ref = FR.logits_ref(w, ocfg, otok, q, texts, r.max_length)
        assert lib.dtype == np.float32 and lib.shape == (15, ocfg.num_labels)
        assert np.abs(lib - ref).max() < 1e-3, (name, float(np.abs(lib - ref).max()))
        docs = [Document(t, {"source": f"s{i}"}) for i, t in enumerate(texts)]
        out = FlashrankRerank(client=r, top_n=15).compress_documents(docs, q)
        # the scores are FlashRank's arithmetic on the library's own logits, bit for bit, in the same order
        want = FR.compress_documents(docs, q, lambda *_: lib, top_n=15)
        assert [d.page_content for d in out] == [t for t, _ in want]
        got_s = np.array([d.metadata["relevance_score"] for d in out], dtype=np.float32)
        want_s = np.array([m["relevance_score"] for _, m in want], dtype=np.float32)
        assert np.array_equal(got_s.view(np.int32), want_s.view(np.int32))
        ref_s = FR.scores(ref)
        bound = _score_bound(ocfg)
        assert np.abs(got_s - ref_s[[d.metadata["id"] for d in out]]).max() <= bound
        _check_order([d.metadata["id"] for d in out], ref_s, bound)


def test_a_document_alone_scores_as_in_a_list_of_fifty(model):
    from ragmeup_b200.flashrank import FlashrankRerank
    r, ocfg, _, _ = model("synthetic:ms-marco-MultiBERT-L-12:3:4.0")
    vocab = synthetic_vocab(ocfg.vocab_size)
    q = synthetic_sentences(vocab, 1, 10, 16, seed=40)[0]
    texts = synthetic_sentences(vocab, 49, 20, 200, seed=41) + synthetic_sentences(vocab, 1, 700, 800, seed=42)
    docs = [Document(t, {}) for t in texts]
    fr = FlashrankRerank(client=r, top_n=50)
    many = {d.metadata["id"]: d.metadata["relevance_score"] for d in fr.compress_documents(docs, q)}
    lib = r.logits(q, texts)
    for i in (0, 17, 49):
        assert np.array_equal(r.logits(q, [texts[i]]).view(np.int32), lib[i:i + 1].view(np.int32)), i
        one = fr.compress_documents([docs[i]], q)[0].metadata["relevance_score"]
        assert np.float32(one).view(np.int32) == np.float32(many[i]).view(np.int32), i


def test_a_call_past_the_token_limit_equals_two_calls(model):
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL
    from ragmeup_b200.flashrank import FlashrankRerank, flashrank_scores
    r, ocfg, _, _ = model("synthetic:ms-marco-TinyBERT-L-2-v2:5:4.0")
    vocab = synthetic_vocab(ocfg.vocab_size)
    q = synthetic_sentences(vocab, 1, 10, 16, seed=50)[0]
    texts = synthetic_sentences(vocab, 300, 500, 800, seed=51)
    cu = r._pairs([q] * 300, texts)[2]
    assert int(cu[-1]) > MAX_TOKENS_PER_CALL and int(cu[150]) < MAX_TOKENS_PER_CALL
    whole = r.logits(q, texts)
    split = np.concatenate([r.logits(q, texts[:150]), r.logits(q, texts[150:])])
    assert np.array_equal(whole.view(np.int32), split.view(np.int32))
    out = FlashrankRerank(client=r, top_n=300).compress_documents([Document(t, {}) for t in texts], q)
    s = flashrank_scores(split)
    assert all(np.float32(d.metadata["relevance_score"]).view(np.int32) == s[d.metadata["id"]].view(np.int32)
               for d in out)


def test_four_threads_on_one_instance_give_the_serial_results(model):
    from ragmeup_b200.flashrank import FlashrankRerank
    r, ocfg, _, _ = model("synthetic:ms-marco-MiniLM-L-12-v2:3:4.0")
    vocab = synthetic_vocab(ocfg.vocab_size)
    fr = FlashrankRerank(client=r, top_n=5)
    calls = [_call_shape(vocab, 60 + 10 * k) for k in range(6)]
    calls = [(q, [Document(t, {"k": k}) for t in texts]) for k, (q, texts) in enumerate(calls)]
    key = lambda out: [(d.page_content, np.float32(d.metadata["relevance_score"]).view(np.int32).item()) for d in out]  # noqa: E731
    serial = [key(fr.compress_documents(docs, q)) for q, docs in calls]
    errors = []

    def worker(tid):
        try:
            for it in range(12):
                k = (tid + it) % 6
                assert key(fr.compress_documents(calls[k][1], calls[k][0])) == serial[k]
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def _snapshot(root, name, seed, scale):
    """write the synthetic MultiBERT shape as a HuggingFace snapshot named as FlashRank's checkpoint"""
    import json
    import os
    from safetensors.numpy import save_file
    from ragmeup_b200.tokenizer import build_wordpiece
    from ragmeup_b200.weights import PRESETS, BertConfig, synthetic_bert_weights
    cfg = BertConfig(**asdict(PRESETS["ms-marco-MultiBERT-L-12"][0]))
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True, scale=scale)
    d = os.path.join(root, name)
    os.makedirs(d)
    save_file({("bert." + k if not k.startswith("classifier") else k): v for k, v in w.items()},
              os.path.join(d, "model.safetensors"))
    json.dump({"vocab_size": cfg.vocab_size, "hidden_size": 768, "num_hidden_layers": 12, "num_attention_heads": 12,
               "intermediate_size": 3072, "max_position_embeddings": 512, "hidden_act": "gelu",
               "id2label": {"0": "LABEL_0", "1": "LABEL_1"}}, open(os.path.join(d, "config.json"), "w"))
    json.dump({"model_max_length": 512}, open(os.path.join(d, "tokenizer_config.json"), "w"))
    open(os.path.join(d, "tokenizer.json"), "w").write(build_wordpiece(synthetic_vocab(cfg.vocab_size)).to_str())
    return bert_ref.BertCfg(**asdict(cfg)), w


def test_ragmeup_default_reranker_wiring(cuda, tmp_path, monkeypatch):
    """ContextualCompressionRetriever(FlashrankRerank(top_n=3), EnsembleRetriever([BM25, Milvus mmr])) as
    RAGHelper builds it with rerank_model=flashrank, against hybrid_ref + flashrank_ref; then rerank provenance"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.flashrank import FlashrankRerank
    from ragmeup_b200.provenance import compute_rerank_provenance
    from ragmeup_b200.retrievers import BM25Retriever, ContextualCompressionRetriever, EnsembleRetriever
    from ragmeup_b200.vectorstore import Milvus
    from ragmeup_b200.weights import resolve_model
    ccfg, cw = _snapshot(str(tmp_path), "amberoad/bert-multilingual-passage-reranking-msmarco", seed=1, scale=4.0)
    monkeypatch.setenv("RAGMEUP_MODEL_DIR", str(tmp_path))
    compressor = FlashrankRerank(top_n=3)                               # RAGHelper.py:480, the default model
    assert compressor.client.config.num_labels == 2 and compressor.client.max_length == 512
    otok = Tokenizer.from_str(compressor.client.tokenizer.to_str())
    o_logits = lambda q, t: FR.logits_ref(cw, ccfg, otok, q, t, 512)    # noqa: E731
    bound = _score_bound(ccfg)

    emb = HuggingFaceEmbeddings(model_name="synthetic:all-MiniLM-L6-v2:0", model_kwargs={"device": "cuda"})
    vocab = synthetic_vocab(30522)
    texts = synthetic_sentences(vocab, 600, 30, 60, seed=17)
    queries = [" ".join(t.split()[3:9]) for t in texts[5:9]]
    documents = [Document(t, {"source": f"f{i % 5}.txt", "id": f"id{i}"}) for i, t in enumerate(texts)]
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="c")
    db.add_documents(documents, ids=[d.metadata["id"] for d in documents])
    sparse = BM25Retriever.from_texts(texts, metadatas=[d.metadata for d in documents])
    dense = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    ensemble = EnsembleRetriever(retrievers=[sparse, dense], weights=[0.5, 0.5])
    rerank = ContextualCompressionRetriever(base_compressor=compressor, base_retriever=ensemble)

    ecfg, ew, *_ = resolve_model(emb.model_name, with_head=False)
    ecfg = bert_ref.BertCfg(**asdict(ecfg))
    X = bert_ref.st_encode(ew, ecfg, emb.tokenizer, texts, "mean", True, 256)
    o_sparse = H.BM25Retriever.from_texts(texts, make_doc=lambda t, m: t)
    by_text = {t: i for i, t in enumerate(texts)}
    for q in queries:
        sp = o_sparse.invoke(q)
        qv = np.asarray(bert_ref.hf_embed_query(ew, ecfg, emb.tokenizer, q, max_seq_length=256), dtype=np.float32)
        de = [texts[r] for r in flat_ref.mmr_search(qv[None], X, 10, "l2", fetch_k=20, lambda_mult=0.5)[0]]
        fused = H.weighted_reciprocal_rank([sp, de], [0.5, 0.5], key=lambda t: t)
        assert [d.page_content for d in ensemble.invoke(q)] == fused
        o_docs = [Document(t, dict(documents[by_text[t]].metadata)) for t in fused]
        ref_scores = FR.scores(o_logits(q, fused))
        want = FR.compress_documents(o_docs, q, lambda *_: o_logits(q, fused), top_n=3)
        out = rerank.invoke(q)
        assert len(out) == 3
        assert [d.metadata["id"] for d in out] == [documents[by_text[d.page_content]].metadata["id"] for d in out]
        got_pos = [fused.index(d.page_content) for d in out]
        assert np.abs(np.array([d.metadata["relevance_score"] for d in out]) - ref_scores[got_pos]).max() <= bound
        srt = np.sort(ref_scores)[::-1]
        if len(fused) == 3 or srt[2] - srt[3] > 2 * bound:              # the oracle's top 3 is unambiguous
            assert sorted(got_pos) == sorted(fused.index(t) for t, _ in want)
        assert all(ref_scores[got_pos[k]] >= ref_scores[got_pos[k + 1]] - 2 * bound for k in range(2))
        # rerank provenance (RAGHelper_local.py:300-308): the reply's documents re-scored against the answer
        answer = " ".join(fused[0].split()[:25])
        oc = FR.FlashrankRerank(o_logits, top_n=3)
        for flag in (None, "True"):
            if flag is None:
                monkeypatch.delenv("attribute_include_query", raising=False)
            else:
                monkeypatch.setenv("attribute_include_query", flag)
            # the reply's documents already carry relevance_score, and their own metadata wins the merge: the
            # scores that come back are the rerank's, unchanged (FlashRank does the same)
            again = compute_rerank_provenance(compressor, q, out, answer)
            assert {d.page_content: d.metadata["relevance_score"] for d in again} == \
                {d.page_content: d.metadata["relevance_score"] for d in out}
            fresh = [Document(d.page_content, dict(documents[by_text[d.page_content]].metadata)) for d in out]
            got = compute_rerank_provenance(compressor, q, fresh, answer)
            ref = P.compute_rerank_provenance(oc, q, fresh, answer, include_query=flag == "True")
            g = {d.page_content: d.metadata["relevance_score"] for d in got}
            r_ = {t: m["relevance_score"] for t, m in ref}
            assert len(got) == 3 and set(g) == set(r_)
            assert max(abs(g[t] - r_[t]) for t in g) <= bound
            assert all(d.metadata["id"] == documents[by_text[d.page_content]].metadata["id"] for d in got)
