"""CPU: the FlashrankRerank drop-in's host logic (ragmeup_b200/flashrank.py) and its oracle (oracle/flashrank_ref.py)
against hand-computed answers, install() registration, FlashRank model resolution and tokenisation of unstripped
pairs.  The device encoder is replaced by a stub that returns chosen logits: only the host side is under test here
(tests/test_flashrank_gpu.py runs the encoder)."""
import json
import os
import sys
import types

import numpy as np
import pytest

from oracle import flashrank_ref as FR
from ragmeup_b200 import flashrank as fl
from ragmeup_b200.documents import Document
from ragmeup_b200.tokenizer import (PairAssembler, RaggedTokenizer, build_wordpiece, load_tokenizer,
                                    synthetic_sentences, synthetic_vocab)
from ragmeup_b200.weights import BertConfig, resolve_flashrank, synthetic_bert_weights

f32 = np.float32


class FixedRanker(fl.Ranker):
    """the product Ranker (rerank, flashrank_scores, sort) with logits given per passage text"""

    def __init__(self, table):
        self.table = table

    def logits(self, query, texts):
        return np.asarray([self.table[t] for t in texts], dtype=f32)


def _docs(texts, metas=None):
    return [Document(t, dict(metas[i]) if metas else {}) for i, t in enumerate(texts)]


def _both(logits, top_n=3, score_threshold=0.0, prefix=""):
    """(product, oracle) results of compress_documents on documents d0..d{n-1} with these logits"""
    texts = [f"d{i}" for i in range(len(logits))]
    table = dict(zip(texts, np.asarray(logits, dtype=f32)))
    got = fl.FlashrankRerank(client=FixedRanker(table), top_n=top_n, score_threshold=score_threshold,
                             prefix_metadata=prefix).compress_documents(_docs(texts), "q")
    want = FR.compress_documents(_docs(texts), "q", lambda q, t: np.asarray([table[x] for x in t]), top_n,
                                 score_threshold, prefix)
    return got, want


# ----------------------------------------------------------------------------------------- the score arithmetic
@pytest.mark.parametrize("fn", [fl.flashrank_scores, FR.scores], ids=["product", "oracle"])
def test_scores_match_hand_computed(fn):
    s = fn(np.array([[0.0], [2.0], [-1.0]], f32))               # one label: sigmoid
    assert s.dtype == f32 and np.allclose(s, [0.5, 0.880797077977882, 0.2689414213699951], rtol=1e-6, atol=0)
    s = fn(np.array([[0.0, 0.0], [0.0, np.log(3.0)], [2.0, -1.0]], f32))   # two labels: softmax column 1
    assert s.dtype == f32 and np.allclose(s, [0.5, 0.75, 1 / (1 + np.e ** 3)], rtol=1e-6, atol=0)
    s = fn(np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0]], f32))   # three labels: still column 1 of the softmax
    e = np.e
    assert np.allclose(s, [1 / 3, e ** 2 / (e + e ** 2 + e ** 3)], rtol=1e-6, atol=0)
    with np.errstate(over="ignore", invalid="ignore"):
        s = fn(np.array([[0.0, 100.0], [100.0, 0.0]], f32))    # exp(100) overflows float32: inf / inf, 1 / inf
    assert np.isnan(s[0]) and s[1] == 0.0


def test_ties_keep_input_order_and_scores_are_float32():
    got, want = _both([[1.0], [3.0], [1.0], [3.0], [1.0]], top_n=5)
    assert [d.metadata["id"] for d in got] == [1, 3, 0, 2, 4] == [m["id"] for _, m in want]
    for d in got:
        assert type(d.metadata["relevance_score"]) is np.float32
    assert got[0].metadata["relevance_score"] == f32(1) / (f32(1) + np.exp(f32(-3)))


def test_top_n_is_cut_before_the_threshold():
    """The passages sort with a NaN among them (two labels, logit 100 on label 1).  Scores, in input order:
    d0 NaN, d1 s(2) = 0.881, d2 s(-3) = 0.047, d3 s(1) = 0.731, d4 s(0) = 0.5.  list.sort(reverse=True) reverses the
    list, sorts it ascending and reverses it back.  The ascending pass over [d4, d3, d2, d1, d0] takes the run
    [d4, d3] and binary-inserts the rest; NaN compares false with everything, so d0 lands last, i.e. FIRST after the
    final reversal: [d0, d1, d3, d4, d2].  [:3] keeps d0, d1, d3 and the threshold then drops d0 (NaN >= 0 is false):
    two documents for top_n = 3.  Thresholding first would give d1, d3, d4."""
    logits = [[0.0, 100.0], [0.0, 2.0], [0.0, -3.0], [0.0, 1.0], [0.0, 0.0]]
    with np.errstate(over="ignore", invalid="ignore"):
        got, want = _both(logits, top_n=3)
    assert [d.metadata["id"] for d in got] == [1, 3] == [m["id"] for _, m in want]
    with np.errstate(over="ignore", invalid="ignore"):
        got, _ = _both(logits, top_n=5, score_threshold=0.6)
    assert [d.metadata["id"] for d in got] == [1, 3]
    got, _ = _both([[0.0, 2.0], [0.0, -3.0], [0.0, 1.0]], top_n=3, score_threshold=0.5)
    assert [d.metadata["id"] for d in got] == [0, 2]                # fewer than top_n without a NaN as well


def test_metadata_merge_and_new_documents():
    texts = ["a", "b", "c"]
    table = {"a": np.array([0.5], f32), "b": np.array([2.0], f32), "c": np.array([-1.0], f32)}
    metas = [{"id": "md5-a", "source": "x"}, {"id": "md5-b", "source": "y"}, {"source": "z"}]
    docs = _docs(texts, metas)
    out = fl.FlashrankRerank(client=FixedRanker(table), top_n=3).compress_documents(docs, "q")
    s = {t: float(fl.flashrank_scores(table[t][None])[0]) for t in texts}
    assert [d.page_content for d in out] == ["b", "a", "c"]
    assert out[0].metadata == {"id": "md5-b", "relevance_score": s["b"], "source": "y"}     # the chunk's own id wins
    assert out[2].metadata == {"id": 2, "relevance_score": s["c"], "source": "z"}           # positional without one
    assert all(d is not o for d in out for o in docs) and docs[1].metadata == metas[1]      # new documents
    out = fl.FlashrankRerank(client=FixedRanker(table), top_n=2, prefix_metadata="fr_").compress_documents(docs, "q")
    assert out[0].metadata == {"fr_id": 1, "fr_relevance_score": s["b"], "id": "md5-b", "source": "y"}
    want = FR.compress_documents(docs, "q", lambda q, t: np.asarray([table[x] for x in t]), 2, 0.0, "fr_")
    assert [(d.page_content, d.metadata) for d in out] == want
    with pytest.raises(ValueError):
        fl.FlashrankRerank(client=FixedRanker(table)).compress_documents([], "q")
    with pytest.raises(TypeError):
        fl.FlashrankRerank(client=FixedRanker(table), cache_folder="/x")        # extra="forbid"
    r = fl.FlashrankRerank(client=FixedRanker(table))
    assert (r.top_n, r.score_threshold, r.model, r.prefix_metadata) == (3, 0.0, None, "")
    assert fl.DEFAULT_MODEL_NAME == "ms-marco-MultiBERT-L-12"


# ----------------------------------------------------------------------------------------- install()
def test_install_registers_flashrank_everywhere_the_reference_imports_it():
    from ragmeup_b200 import install
    c = install.install()
    from langchain.retrievers.document_compressors import FlashrankRerank as A
    from langchain_community.document_compressors import FlashrankRerank as B
    from langchain_community.document_compressors.flashrank_rerank import FlashrankRerank as C
    assert A is B is C is c["FlashrankRerank"] is fl.FlashrankRerank
    from langchain.retrievers import ContextualCompressionRetriever, EnsembleRetriever  # still there
    assert ContextualCompressionRetriever is c["ContextualCompressionRetriever"] and EnsembleRetriever


def test_rebased_class_on_stub_langchain(monkeypatch):
    pydantic = pytest.importorskip("pydantic")

    class Embeddings:
        pass

    class VectorStore:
        @property
        def embeddings(self):
            return None

        def as_retriever(self, **kw):
            return ("lc-retriever", self, kw)

    class BaseDocumentCompressor(pydantic.BaseModel):
        pass

    class BaseRetriever(pydantic.BaseModel):
        pass

    mods = {
        "langchain_core": types.ModuleType("langchain_core"),
        "langchain_core.embeddings": types.SimpleNamespace(Embeddings=Embeddings),
        "langchain_core.vectorstores": types.SimpleNamespace(VectorStore=VectorStore),
        "langchain_core.documents": types.SimpleNamespace(BaseDocumentCompressor=BaseDocumentCompressor, Document=Document),
        "langchain_core.retrievers": types.SimpleNamespace(BaseRetriever=BaseRetriever),
    }
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    from ragmeup_b200 import install
    cls = install.build_classes()["FlashrankRerank"]
    assert issubclass(cls, BaseDocumentCompressor) and cls.__name__ == "FlashrankRerank"
    table = {"a": np.array([0.0, 1.0], f32), "b": np.array([0.0, 2.0], f32)}
    r = cls(client=FixedRanker(table), top_n=1, prefix_metadata="p_")
    assert (r.top_n, r.score_threshold, r.model, r.prefix_metadata) == (1, 0.0, None, "p_")
    out = r.compress_documents(_docs(["a", "b"]), "q")
    assert [d.page_content for d in out] == ["b"] and out[0].metadata["p_id"] == 1
    with pytest.raises(pydantic.ValidationError):
        cls(client=FixedRanker(table), top_k=3)                               # extra="forbid"


# ----------------------------------------------------------------------------------------- model resolution
HF_CFG = {"vocab_size": 400, "hidden_size": 128, "num_hidden_layers": 1, "num_attention_heads": 2,
          "intermediate_size": 256, "max_position_embeddings": 512, "hidden_act": "gelu"}


def _snapshot(d, labels=1, cfg_labels="same", fmt="safetensors", tokenizer_max=None, extra_cfg=None, seed=1):
    """a small BERT cross-encoder snapshot at directory d; returns its weights"""
    os.makedirs(d, exist_ok=True)
    cfg = BertConfig(vocab_size=400, hidden=128, layers=1, heads=2, ffn=256, max_pos=512, num_labels=labels)
    w = synthetic_bert_weights(cfg, seed=seed, with_head=True)
    c = dict(HF_CFG, **(extra_cfg or {}))
    n = labels if cfg_labels == "same" else cfg_labels
    if n is not None:
        c["id2label"] = {str(i): f"LABEL_{i}" for i in range(n)}
    json.dump(c, open(os.path.join(d, "config.json"), "w"))
    if fmt == "safetensors":
        from safetensors.numpy import save_file
        save_file({"bert." + k if not k.startswith("classifier") else k: v for k, v in w.items()},
                  os.path.join(d, "model.safetensors"))
    else:
        import torch
        sd = {("bert." + k if not k.startswith("classifier") else k): torch.from_numpy(v) for k, v in w.items()}
        sd["bert.embeddings.position_ids"] = torch.arange(512)[None]             # an integer buffer, as old files hold
        torch.save(sd, os.path.join(d, "pytorch_model.bin"))
    if tokenizer_max is not None:
        json.dump({"model_max_length": tokenizer_max, "do_lower_case": True},
                  open(os.path.join(d, "tokenizer_config.json"), "w"))
    open(os.path.join(d, "tokenizer.json"), "w").write(build_wordpiece(synthetic_vocab(400)).to_str())
    return w


def test_both_name_forms_resolve(tmp_path, monkeypatch):
    monkeypatch.delenv("RAGMEUP_MODEL_DIR", raising=False)
    w = _snapshot(str(tmp_path / "a" / "ms-marco-TinyBERT-L-2-v2"))
    cfg, got, max_len, src = resolve_flashrank("ms-marco-TinyBERT-L-2-v2", cache_folder=str(tmp_path / "a"))
    assert src == str(tmp_path / "a" / "ms-marco-TinyBERT-L-2-v2") and cfg.num_labels == 1
    assert all(np.array_equal(got[k], w[k]) for k in w)
    _snapshot(str(tmp_path / "b" / "amberoad" / "bert-multilingual-passage-reranking-msmarco"), labels=2)
    monkeypatch.setenv("RAGMEUP_MODEL_DIR", str(tmp_path / "b"))
    cfg, got, max_len, src = resolve_flashrank("ms-marco-MultiBERT-L-12")
    assert src.endswith("amberoad/bert-multilingual-passage-reranking-msmarco") and cfg.num_labels == 2
    _snapshot(str(tmp_path / "b" / "ms-marco-MiniLM-L-12-v2"))
    assert resolve_flashrank("ms-marco-MiniLM-L-12-v2")[3] == str(tmp_path / "b" / "ms-marco-MiniLM-L-12-v2")
    with pytest.raises(FileNotFoundError) as e:
        resolve_flashrank("ms-marco-TinyBERT-L-2-v2")
    assert "ms-marco-TinyBERT-L-2-v2" in str(e.value) and "cross-encoder/ms-marco-TinyBERT-L-2-v2" in str(e.value)


@pytest.mark.parametrize("name", ["rank-T5-flan", "rank_zephyr_7b_v1_full", "ce-esci-MiniLM-L12-v2-typo", "bert-base"])
def test_other_flashrank_names_are_refused(name):
    with pytest.raises(ValueError) as e:
        resolve_flashrank(name)
    assert "ms-marco-MultiBERT-L-12" in str(e.value) and "ms-marco-TinyBERT-L-2-v2" in str(e.value)


def test_pytorch_bin_snapshot_loads_the_safetensors_arrays(tmp_path):
    w = _snapshot(str(tmp_path / "st" / "ms-marco-MiniLM-L-12-v2"), labels=2)
    _snapshot(str(tmp_path / "pt" / "ms-marco-MiniLM-L-12-v2"), labels=2, fmt="bin")
    assert not os.path.exists(tmp_path / "pt" / "ms-marco-MiniLM-L-12-v2" / "model.safetensors")
    a = resolve_flashrank("ms-marco-MiniLM-L-12-v2", cache_folder=str(tmp_path / "st"))
    b = resolve_flashrank("ms-marco-MiniLM-L-12-v2", cache_folder=str(tmp_path / "pt"))
    assert a[0] == b[0] and a[2] == b[2]
    for k in w:
        assert b[1][k].dtype == np.float32 and np.array_equal(a[1][k], b[1][k]) and np.array_equal(b[1][k], w[k]), k


def test_labels_come_from_the_classifier_and_must_agree_with_the_config(tmp_path):
    _snapshot(str(tmp_path / "x" / "ms-marco-MultiBERT-L-12"), labels=2, cfg_labels=1)
    with pytest.raises(ValueError, match="2 rows"):
        resolve_flashrank("ms-marco-MultiBERT-L-12", cache_folder=str(tmp_path / "x"))
    _snapshot(str(tmp_path / "y" / "ms-marco-MultiBERT-L-12"), labels=2, cfg_labels=None)   # config silent: 2 rows
    assert resolve_flashrank("ms-marco-MultiBERT-L-12", cache_folder=str(tmp_path / "y"))[0].num_labels == 2


@pytest.mark.parametrize("tokenizer_max,want", [(None, 512), (128, 128), (512, 512), (1000000000000000019884624838656, 512)])
def test_max_length_follows_tokenizer_config(tmp_path, tokenizer_max, want):
    d = str(tmp_path / "ms-marco-TinyBERT-L-2-v2")
    _snapshot(d, tokenizer_max=tokenizer_max)
    json.dump({"max_seq_length": 48}, open(os.path.join(d, "sentence_bert_config.json"), "w"))   # not FlashRank's
    assert resolve_flashrank("ms-marco-TinyBERT-L-2-v2", cache_folder=str(tmp_path))[2] == want
    assert resolve_flashrank("ms-marco-TinyBERT-L-2-v2", cache_folder=str(tmp_path), max_length=100)[2] == min(want, 100)


def test_synthetic_presets_have_the_flashrank_shapes():
    cfg, w, max_len, src = resolve_flashrank("synthetic:ms-marco-MultiBERT-L-12:0")
    assert (cfg.vocab_size, cfg.hidden, cfg.heads, cfg.ffn, cfg.layers, cfg.num_labels) == (105879, 768, 12, 3072, 12, 2)
    assert w["embeddings.word_embeddings.weight"].shape == (105879, 768) and max_len == 512 and src is None
    cfg = resolve_flashrank("synthetic:ms-marco-TinyBERT-L-2-v2")[0]
    assert (cfg.hidden, cfg.heads, cfg.head_dim, cfg.ffn, cfg.layers, cfg.num_labels) == (128, 2, 64, 512, 2, 1)
    cfg = resolve_flashrank("synthetic:ms-marco-MiniLM-L-12-v2")[0]
    assert (cfg.hidden, cfg.heads, cfg.ffn, cfg.layers, cfg.num_labels) == (384, 12, 1536, 12, 1)
    v = synthetic_vocab(105879)
    assert len(v) == 105879 and sorted(v.values()) == list(range(105879))
    # the smaller synthetic vocabularies every other test and the benchmark use are the ones they always were
    import hashlib
    for n, digest in ((1000, "62cf1e5e8de8c16fd0dab96ab2d4b235175a6515232a988e734b78daa6ccb549"),
                      (30522, "87a1a4cbca5902bdb9af6bfa3790d32d51909843fa2323a30f4e63a5592d62a6")):
        v = synthetic_vocab(n)
        assert hashlib.sha256("\n".join(sorted(v, key=v.get)).encode()).hexdigest() == digest, n


# ----------------------------------------------------------------------------------------- tokenisation
PADS = [" ", "  \t", "\n", "\r\n", "\t \n ", "\xa0", "　", " ", "\x85", "\x0b\x0c", "\x1f", "   "]


def _padded(texts, seed):
    rng = np.random.default_rng(seed)
    return [PADS[int(rng.integers(len(PADS)))] + t + PADS[int(rng.integers(len(PADS)))] for t in texts]


@pytest.mark.parametrize("kind", ["tokenizer.json", "vocab.txt"])
@pytest.mark.parametrize("max_length", [512, 64])
def test_unstripped_pairs_tokenise_like_stripped_ones(tmp_path, kind, max_length):
    vocab = synthetic_vocab(30522)
    if kind == "tokenizer.json":
        open(tmp_path / "tokenizer.json", "w").write(build_wordpiece(vocab).to_str())
    else:
        with open(tmp_path / "vocab.txt", "w", encoding="utf-8") as f:
            f.write("\n".join(sorted(vocab, key=vocab.get)) + "\n")
    tok = load_tokenizer(str(tmp_path), 30522)
    docs = synthetic_sentences(vocab, 60, 100, 160, seed=3) + synthetic_sentences(vocab, 20, 400, 700, seed=4)
    queries = synthetic_sentences(vocab, 80, 5, 20, seed=5)
    docs, queries = docs + ["", "x"], queries + ["q", ""]
    rq, rd = _padded(queries, 6), _padded(docs, 7)
    assert all(a != a.strip() for a in rq) and all(a != a.strip() for a in rd)
    stripped = RaggedTokenizer(tok, max_length)([q.strip() for q in rq], [d.strip() for d in rd])
    raw = RaggedTokenizer(tok, max_length)(rq, rd)
    assembled = PairAssembler(tok, max_length)(rq, rd)
    for x, y, z in zip(stripped, raw, assembled):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    lens = np.diff(stripped[2])
    assert lens.max() == max_length and (lens == max_length).sum() >= 10          # truncated pairs are covered


class StubEncoder:
    """records what the product sends to the device and returns logits derived from it"""
    calls = []

    def __init__(self, cfg, w, with_head):
        self.cfg = cfg

    def classify_host(self, ids, typ, cu):
        StubEncoder.calls.append((ids.copy(), typ.copy(), cu.copy()))
        L = self.cfg.num_labels
        return np.asarray([[(int(ids[cu[b]:cu[b + 1]].sum()) % 97 - 48) / 8.0 + j for j in range(L)]
                           for b in range(len(cu) - 1)], dtype=f32)


def test_product_ranker_tokenises_unstripped_text_at_flashranks_max_length(tmp_path, monkeypatch):
    """the Ranker built from a snapshot: pairs at tokenizer_config's model_max_length, texts as given, FlashRank's
    activation even though the config names another one"""
    d = str(tmp_path / "ms-marco-TinyBERT-L-2-v2")
    _snapshot(d, tokenizer_max=64, extra_cfg={"sbert_ce_default_activation_function": "torch.nn.modules.linear.Identity"})
    monkeypatch.setattr(fl, "BertEncoder", StubEncoder)
    StubEncoder.calls = []
    r = fl.FlashrankRerank(client=fl.Ranker("ms-marco-TinyBERT-L-2-v2", cache_dir=str(tmp_path)), top_n=4)
    assert r.client.max_length == 64
    vocab = synthetic_vocab(400)
    texts = _padded(synthetic_sentences(vocab, 6, 20, 80, seed=1), 2)
    q = " \t" + synthetic_sentences(vocab, 1, 5, 9, seed=3)[0] + "\n"
    out = r.compress_documents(_docs(texts), q)
    ids, typ, cu = StubEncoder.calls[-1]
    want = RaggedTokenizer(load_tokenizer(d), 64)([q.strip()] * 6, [t.strip() for t in texts])
    assert np.array_equal(ids, want[0]) and np.array_equal(typ, want[1]) and np.array_equal(cu, want[2])
    logits = StubEncoder(r.client.config, None, True).classify_host(ids, typ, cu)
    ranked = FR.rerank(q, [{"id": i, "text": t, "meta": {}} for i, t in enumerate(texts)], lambda *_: logits)[:4]
    assert [d.page_content for d in out] == [p["text"] for p in ranked]       # texts come back unstripped
    assert [d.metadata["relevance_score"] for d in out] == [p["score"] for p in ranked]
    assert all(0 < p["score"] < 1 for p in ranked)                            # sigmoid, not the config's identity


def test_construction_without_cuda_raises():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from ragmeup_b200 import _lib
    with pytest.raises(_lib.RmuError):
        fl.Ranker("synthetic:ms-marco-TinyBERT-L-2-v2")
    with pytest.raises(_lib.RmuError):
        fl.FlashrankRerank(model="synthetic:ms-marco-TinyBERT-L-2-v2", top_n=3)
