"""GPU: X-MOD on the encoder (the language adapter after each layer's FFN output) and ColBERT-XM.  The whole stack
against the float64 forward on the split weights (oracle/xmod_ref.py) at the tiny-xmod and xmod-base shapes, with the
CLS-row last layer bit-identical to the full one through the heads; the language selection; then the product:
HuggingFaceCrossEncoder on colbert-xm against the ColBERT oracle, RAGMeUp's rerank retriever on a ColBERT-XM snapshot,
and X-MOD snapshots as an embedder and as a cross-encoder.  Bounds follow tests/test_xlmr_gpu.py (u = 2^-24)."""
import json
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref, colbert_ref
from oracle import encoder_kernels_ref as ref
from oracle import xmod_ref
from ragmeup_b200 import weights as W
from ragmeup_b200.weights import PRESETS, XmodConfig, synthetic_bert_weights, synthetic_colbert

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


@pytest.fixture(autouse=True)
def _no_tf32_no_language_env(monkeypatch):
    monkeypatch.delenv(W.XMOD_LANGUAGE_ENV, raising=False)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _cfg(preset, **kw):
    return XmodConfig(**{**asdict(PRESETS[preset][0]), **kw})


def _w32(wd):
    """the fp32 forward's weights: every weight the encoder holds as split planes, as hi + lo"""
    return {k: ref.split_weight(v).float() if k.endswith(xmod_ref.GEMM_WEIGHTS) else v for k, v in wd.items()}


# -------------------------------------------------------------------------------------------------- whole stack
FLOOR = 4.0
OUTPUTS = ("hidden", "mean", "mean_norm", "cls", "cls_norm", "logits")
# (preset, weight scale, language, lengths, c, c_mean): the rule of test_xlmr_stack_matches_float64_forward
STACK = {
    "xmod-base": ("xmod-base", 1.0, "de_DE", [0, 1, 9, 16, 129, 0, 255, 256, 257, 384, 512, 0], 90, 150),
    "xmod-base x4": ("xmod-base", 4.0, "fr_XX", [1, 17, 0, 300, 512], 90, 150),
    "tiny-xmod": ("tiny-xmod", 1.0, "fr_XX", [0, 1, 9, 16, 127, 128, 0, 64], 90, 150),
    "tiny-xmod x4": ("tiny-xmod", 4.0, "en_XX", [0, 1, 9, 128, 0, 33, 128], 90, 150),
}


def _batch(lens, vocab, seed):
    rng = np.random.default_rng(seed)
    seqs = []
    for n in lens:
        s = np.r_[0, rng.integers(5, vocab - 1, max(n - 2, 0)), 2][:n]
        if n > 6:
            s[n // 2] = 1                             # a literal <pad> inside the text
        seqs.append(s)
    ids = np.concatenate(seqs + [np.zeros(0, np.int64)]).astype(np.int32)
    return ids, np.r_[0, np.cumsum(lens)].astype(np.int32), max(lens)


def _gpu(enc, ids, cu, mx):
    out = {"hidden": enc.hidden_tokens(ids, None, cu, mx), "logits": enc.classify_tokens(ids, None, cu, mx)}
    for mode in ("mean", "cls"):
        out[mode] = enc.embed_tokens(ids, None, cu, mx, mode, False)
        out[mode + "_norm"] = enc.embed_tokens(ids, None, cu, mx, mode, True)
    torch.cuda.synchronize()
    return out


def _fp32(w32, cfg, ids, cu):
    lens = np.diff(cu)
    ocfg = xmod_ref.XmodCfg(**asdict(cfg))
    H = cfg.hidden
    out = {k: [] for k in OUTPUTS}
    with torch.no_grad():
        for b, n in enumerate(lens):
            if n == 0:
                z = torch.zeros((1, H), device="cuda")
                for k in ("mean", "mean_norm", "cls", "cls_norm"):
                    out[k].append(z)
                out["logits"].append(xmod_ref.classifier_head(w32, z[:, None, :]))
                continue
            I = torch.from_numpy(ids[cu[b]:cu[b + 1]].astype(np.int64))[None]
            h = xmod_ref.xmod_encoder_forward(w32, ocfg, I, torch.ones_like(I), device="cuda")
            mask = torch.ones_like(I).cuda()
            out["hidden"].append(h[0])
            for mode in ("mean", "cls"):
                e = bert_ref.pool(h, mask, mode)
                out[mode].append(e)
                out[mode + "_norm"].append(bert_ref.l2_normalize(e))
            out["logits"].append(xmod_ref.classifier_head(w32, h))
    return {k: torch.cat(v).double() for k, v in out.items()}


def _split_heads(enc, w, ids, cu, mx):
    """rmu_encoder_hidden -> split planes -> rmu_debug_cls_head / rmu_debug_pool (CLS)"""
    L = _lib()
    lib = L.lib()
    H, nl, B = enc.cfg.hidden, enc.cfg.num_labels, len(cu) - 1
    h = enc.hidden_tokens(ids, None, cu, mx)
    hi = torch.empty(h.shape, dtype=torch.float16, device="cuda")
    lo = torch.empty_like(hi)
    L.check(lib.rmu_debug_split_planes(h.data_ptr(), h.numel(), hi.data_ptr(), lo.data_ptr(), L.stream_ptr()), "split")
    cu_d = _i32(cu)
    head = {k: torch.from_numpy(w[k]).cuda() for k in ("pooler.dense.weight", "pooler.dense.bias", "classifier.weight",
                                                        "classifier.bias")}
    logits = torch.empty((B, nl), dtype=torch.float32, device="cuda")
    L.check(lib.rmu_debug_cls_head(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, nl,
                                   head["pooler.dense.weight"].data_ptr(), head["pooler.dense.bias"].data_ptr(),
                                   head["classifier.weight"].data_ptr(), head["classifier.bias"].data_ptr(),
                                   logits.data_ptr(), L.stream_ptr()), "cls_head")
    emb = {}
    for norm in (0, 1):
        e = torch.empty((B, H), dtype=torch.float32, device="cuda")
        L.check(lib.rmu_debug_pool(hi.data_ptr(), lo.data_ptr(), cu_d.data_ptr(), B, H, 1, norm, e.data_ptr(),
                                   L.stream_ptr()), "pool")
        emb[norm] = e
    torch.cuda.synchronize()
    return logits, emb


def _compare(got, want, f32, cu, c_rest, c_mean, outputs=OUTPUTS):
    nonempty = torch.from_numpy(np.diff(cu) > 0).cuda()
    report, fails = [], []
    for name in outputs:
        g, w_, f = got[name].double(), want[name], f32[name]
        assert torch.isfinite(g).all(), name
        c = c_mean if name.startswith("mean") else c_rest
        rows = slice(None) if name in ("hidden", "logits") else nonempty
        d = (g - w_).abs(); e = (f[rows] - w_[rows]).abs()
        gmax, grms, fmax, frms = float(d.max()), float(d.pow(2).mean().sqrt()), float(e.max()), float(e.pow(2).mean().sqrt())
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {gmax / fmax:.3g}, rms {grms:.3g} / {frms:.3g} = "
                      f"{grms / frms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(report[-1])
    return report, fails


@pytest.mark.parametrize("case", list(STACK))
def test_xmod_stack_matches_float64_forward(cuda, case):
    from ragmeup_b200.encoder import BertEncoder
    preset, scale, lang, lens, c_rest, c_mean = STACK[case]
    cfg = _cfg(preset, language=lang)
    w = synthetic_bert_weights(cfg, seed=19, with_head=True, scale=scale)
    enc = BertEncoder(cfg, w, with_head=True)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    ids, cu, mx = _batch(lens, cfg.vocab_size, 9)
    got = _gpu(enc, ids, cu, mx)
    want = xmod_ref.xmod_stack_ref(wd, cfg, ids, cu, "split", device="cuda")
    f32 = _fp32(_w32(wd), cfg, ids, cu)
    report, fails = _compare(got, want, f32, cu, c_rest, c_mean)
    print(f"\nX-MOD stack {case}:\n  " + "\n  ".join(report))
    nonempty = torch.from_numpy(np.diff(cu) > 0).cuda()
    for name in ("mean", "cls"):
        assert (got[name][~nonempty] == 0).all()
    assert not fails, f"{case}: beyond {c_rest} (means {c_mean}) x fp32's error: " + "; ".join(fails)
    # the CLS-row last layer: logits and CLS embeddings are the last hidden state's through the heads, bit for bit
    logits, emb = _split_heads(enc, w, ids, cu, mx)
    assert torch.equal(logits, got["logits"]), "logits differ from the heads on rmu_encoder_hidden"
    assert torch.equal(emb[0] + 0.0, got["cls"] + 0.0) and torch.equal(emb[1] + 0.0, got["cls_norm"] + 0.0)
    # host entry points equal the device ones; the longest sequence alone equals its rows in the batch
    assert np.array_equal(enc.classify_host(ids, None, cu), got["logits"].cpu().numpy())
    assert np.array_equal(enc.embed_host(ids, None, cu, "cls", True), got["cls_norm"].cpu().numpy())
    assert np.array_equal(enc.embed_host(ids, None, cu, "mean", True), got["mean_norm"].cpu().numpy())
    b = int(np.argmax(np.diff(cu)))
    t0, t1 = int(cu[b]), int(cu[b + 1])
    one = _gpu(enc, ids[t0:t1], np.array([0, t1 - t0], np.int32), t1 - t0)
    assert torch.equal(one["hidden"], got["hidden"][t0:t1]) and torch.equal(one["logits"][0], got["logits"][b])


def test_the_language_selects_the_adapter(cuda):
    """one weight set, an encoder per language: the outputs differ, and each equals the oracle of its own language"""
    from ragmeup_b200.encoder import BertEncoder
    cfg = _cfg("tiny-xmod")
    w = synthetic_bert_weights(cfg, seed=23, with_head=True, scale=2.0)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    ids, cu, mx = _batch([1, 9, 40, 128, 77], cfg.vocab_size, 4)
    got = {}
    for lang in cfg.languages:
        c = _cfg("tiny-xmod", language=lang)
        got[lang] = _gpu(BertEncoder(c, w, with_head=True), ids, cu, mx)
        want = xmod_ref.xmod_stack_ref(wd, c, ids, cu, "split", device="cuda")
        report, fails = _compare(got[lang], want, _fp32(_w32(wd), c, ids, cu), cu, 90, 150)
        print(f"\nX-MOD {lang}:\n  " + "\n  ".join(report))
        assert not fails, f"{lang}: " + "; ".join(fails)
    for a, b in (("en_XX", "de_DE"), ("de_DE", "fr_XX")):
        assert float((got[a]["hidden"] - got[b]["hidden"]).abs().max()) > 1e-2
        assert float((got[a]["logits"] - got[b]["logits"]).abs().max()) > 1e-4


# -------------------------------------------------------------------------------------------------------- ColBERT-XM
@pytest.fixture(scope="module")
def scorers(cuda):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    return {n: HuggingFaceCrossEncoder(model_name=n) for n in ("synthetic:colbert-xm:1", "synthetic:colbert-xm:1:4",
                                                               "synthetic:tiny-colbert-xm:2")}


def _texts(tok, n, lo, hi, seed):
    words = sorted(p[1:] for p in tok.get_vocab() if p.startswith("▁") and len(p) > 2)
    rng = np.random.default_rng(seed)
    return [" ".join(words[int(j)] for j in rng.integers(0, len(words), int(rng.integers(lo, hi + 1)))) for _ in range(n)]


BOUND = 1e-3


@pytest.mark.parametrize("name", ["synthetic:colbert-xm:1", "synthetic:colbert-xm:1:4"])
@pytest.mark.parametrize("shape", ["ragmeup", "bulk", "long"])
def test_colbert_xm_score_matches_oracle(scorers, name, shape):
    from ragmeup_b200.tokenizer import load_tokenizer
    ce = scorers[name]
    tok = ce.colbert.tokenizer._tok
    if shape == "ragmeup":
        q = _texts(tok, 1, 5, 12, 1)[0]
        pairs = [(q, d) for d in _texts(tok, 14, 60, 120, 2)]
    elif shape == "bulk":
        qs, ds = _texts(tok, 5, 3, 40, 3) + ["", "?"], _texts(tok, 40, 1, 150, 4) + ["", ". , ;", "<pad> x"]
        rng = np.random.default_rng(5)
        pairs = [(qs[int(rng.integers(len(qs)))], ds[int(rng.integers(len(ds)))]) for _ in range(100)]
    else:
        pairs = [(q, d) for q, d in zip(_texts(tok, 3, 40, 60, 6), _texts(tok, 3, 250, 400, 7))]
    got = ce.score(pairs)
    parts = name.split(":")
    cfg, w, lin, spec = synthetic_colbert(parts[1], int(parts[2]), float(parts[3]) if len(parts) > 3 else 1.0)
    want = xmod_ref.score_pairs(w, cfg, lin, spec, load_tokenizer(None, cfg.vocab_size, xlmr=True), pairs, device="cuda")
    assert got.dtype == np.float32 and got.shape == (len(pairs),)
    err = float(np.abs(got - want).max())
    print(f"\n{name} {shape}: max |score - oracle| = {err:.3g}")
    assert err <= BOUND
    assert torch.equal(ce.score_tensor(pairs).cpu(), torch.from_numpy(got))


def test_colbert_xm_vectors_match_float64(scorers):
    """token vectors of queries (key-limited [MASK] padding) and documents against the float64 stack"""
    sc = scorers["synthetic:tiny-colbert-xm:2"].colbert
    cfg, w, lin, spec = synthetic_colbert("tiny-colbert-xm", 2)
    tok = sc.tokenizer._tok
    qids, qcu, nk = sc.tokenizer.queries(_texts(tok, 3, 1, 20, 8))
    dids, dcu, keep = sc.tokenizer.docs(_texts(tok, 4, 1, 90, 9))
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    ld = torch.from_numpy(lin).cuda()
    for ids, cu, n, k in ((qids, qcu, nk, None), (dids, dcu, None, keep)):
        got = sc.vectors_tensor(ids, cu, n, k).double()
        want = xmod_ref.colbert_stack_ref(wd, cfg, ld, ids, cu, n, k, "split", device="cuda")["vectors"]
        err = float((got - want).abs().max())
        print(f"\nColBERT-XM vectors: max |err| = {err:.3g}")
        assert err < 1e-5


def test_colbert_xm_past_the_token_limit_equals_two_calls(scorers):
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL
    ce = scorers["synthetic:tiny-colbert-xm:2"]
    tok = ce.colbert.tokenizer._tok
    L = ce.colbert.spec.doc_maxlen
    n = MAX_TOKENS_PER_CALL // L + 3
    base = _texts(tok, 50, 80, 90, 100)
    docs = [f"doc {i} " + base[i % 50] for i in range(n)]
    assert int(ce.colbert.tokenizer.docs(docs)[1][-1]) > MAX_TOKENS_PER_CALL
    q = _texts(tok, 2, 4, 9, 8)
    pairs = [(q[i % 2], d) for i, d in enumerate(docs)]
    whole = ce.score(pairs)
    h = len(pairs) // 2
    assert np.array_equal(whole, np.concatenate([ce.score(pairs[:h]), ce.score(pairs[h:])]))
    assert torch.equal(ce.score_tensor(pairs).cpu(), torch.from_numpy(whole))


# ------------------------------------------------------------------------------------------------------ snapshots
def _conf(cfg, **kw):
    d = {"model_type": "xmod", "vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden,
         "num_hidden_layers": cfg.layers, "num_attention_heads": cfg.heads, "intermediate_size": cfg.ffn,
         "max_position_embeddings": cfg.max_pos, "type_vocab_size": 1, "layer_norm_eps": cfg.ln_eps, "pad_token_id": 1,
         "adapter_reduction_factor": cfg.hidden // cfg.adapter_dim, "languages": list(cfg.languages),
         "default_language": "de_DE", "pre_norm": False, "adapter_layer_norm": False, "adapter_reuse_layer_norm": True,
         "ln_before_adapter": True}
    d.update(kw)
    return d


def _write(path, conf, tensors, tok, meta=None):
    from safetensors.numpy import save_file
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(conf, f)
    save_file(tensors, os.path.join(path, "model.safetensors"))
    tok.save(os.path.join(path, "tokenizer.json"))
    if meta is not None:
        with open(os.path.join(path, "artifact.metadata"), "w") as f:
            json.dump(meta, f)
    return str(path)


def test_ragmeup_rerank_retriever_on_a_colbert_xm_snapshot(cuda, tmp_path, monkeypatch):
    """ContextualCompressionRetriever(ScoredCrossEncoderReranker(HuggingFaceCrossEncoder("antoinelouis/colbert-xm"),
    top_n=3), EnsembleRetriever([BM25, Milvus mmr])) on a snapshot of ColBERT-XM's layout"""
    from oracle import flat_ref
    from oracle import hybrid_ref as HR
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.documents import Document
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.retrievers import BM25Retriever, ContextualCompressionRetriever, EnsembleRetriever
    from ragmeup_b200.tokenizer import load_tokenizer
    from ragmeup_b200.vectorstore import Milvus
    from ragmeup_b200.weights import resolve_model
    cfg, w, lin, _ = synthetic_colbert("tiny-colbert-xm", 3, 4.0)
    tok = load_tokenizer(None, cfg.vocab_size, xlmr=True)
    meta = {"query_maxlen": 24, "doc_maxlen": 100, "dim": 128, "similarity": "cosine", "attend_to_mask_tokens": False,
            "query_token_id": "[unused0]", "doc_token_id": "[unused1]"}
    snap = _write(tmp_path / "antoinelouis" / "colbert-xm", _conf(cfg, architectures=["HF_ColBERT"]),
                  {**{"roberta." + k: v for k, v in w.items()}, "linear.weight": lin}, tok, meta)
    monkeypatch.setenv("RAGMEUP_MODEL_DIR", str(tmp_path))
    ce = HuggingFaceCrossEncoder(model_name="antoinelouis/colbert-xm")
    assert ce.colbert is not None and ce.config.language == "de_DE" and ce.colbert.spec.doc_maxlen == 100
    spec = ce.colbert.spec
    ocfg = XmodConfig(**{**asdict(cfg), "language": "de_DE"})
    compressor = ScoredCrossEncoderReranker(model=ce, top_n=3)

    emb = HuggingFaceEmbeddings(model_name="synthetic:all-MiniLM-L6-v2:0", model_kwargs={"device": "cuda"})
    texts = _texts(tok, 300, 30, 60, 17)
    queries = [" ".join(t.split()[3:9]) for t in texts[5:8]]
    documents = [Document(t, {"source": f"f{i % 5}.txt", "id": f"id{i}"}) for i, t in enumerate(texts)]
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="xm")
    db.add_documents(documents, ids=[d.metadata["id"] for d in documents])
    sparse = BM25Retriever.from_texts(texts, metadatas=[d.metadata for d in documents])
    dense = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    rerank = ContextualCompressionRetriever(base_compressor=compressor,
                                            base_retriever=EnsembleRetriever(retrievers=[sparse, dense], weights=[0.5, 0.5]))
    ecfg, ew, *_ = resolve_model(emb.model_name, with_head=False)
    ecfg = bert_ref.BertCfg(**asdict(ecfg))
    X = bert_ref.st_encode(ew, ecfg, emb.tokenizer, texts, "mean", True, 256)
    o_sparse = HR.BM25Retriever.from_texts(texts, make_doc=lambda t, m: t)
    for q in queries:
        sp = o_sparse.invoke(q)
        qv = np.asarray(bert_ref.hf_embed_query(ew, ecfg, emb.tokenizer, q, max_seq_length=256), dtype=np.float32)
        de = [texts[r] for r in flat_ref.mmr_search(qv[None], X, 10, "l2", fetch_k=20, lambda_mult=0.5)[0]]
        fused = HR.weighted_reciprocal_rank([sp, de], [0.5, 0.5], key=lambda t: t)
        want = xmod_ref.score_pairs(w, ocfg, lin, spec, tok, [(q, t) for t in fused], device="cuda")
        out = rerank.invoke(q)
        assert len(out) == 3
        got = np.array([d.metadata["relevance_score"] for d in out])
        pos = [fused.index(d.page_content) for d in out]
        assert np.abs(got - want[pos]).max() <= BOUND
        order = np.argsort(-want, kind="stable")
        assert all(want[p] >= want[order[2]] - 2 * BOUND for p in pos)


def _hf_batch(tok, a, b, max_length):
    t = colbert_ref._copy(tok)
    t.enable_truncation(max_length=max_length, strategy="longest_first")
    t.enable_padding(pad_id=1, pad_token="<pad>")
    enc = t.encode_batch(list(a) if b is None else list(zip(a, b)))
    return (torch.tensor([e.ids for e in enc], dtype=torch.long), torch.tensor([e.attention_mask for e in enc],
                                                                                dtype=torch.long))


def test_xmod_snapshot_as_embedder_and_cross_encoder(cuda, tmp_path):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.tokenizer import load_tokenizer
    cfg = _cfg("tiny-xmod", language="de_DE")
    ocfg = xmod_ref.XmodCfg(**asdict(cfg))
    tok = load_tokenizer(None, cfg.vocab_size, xlmr=True)
    texts = _texts(tok, 20, 1, 80, 31) + [""]
    # an embedder: bare tensor names, as XmodModel.save_pretrained writes them
    we = synthetic_bert_weights(cfg, seed=6, scale=2.0)
    p = _write(tmp_path / "xmod-emb", _conf(cfg), we, tok)
    emb = HuggingFaceEmbeddings(model_name=p, encode_kwargs={"normalize_embeddings": True})
    assert isinstance(emb.config, XmodConfig) and emb.config.language == "de_DE"
    got = np.asarray(emb.embed_documents(texts))
    ids, mask = _hf_batch(tok, [t.strip() for t in texts], None, emb.max_seq_length)
    with torch.no_grad():
        want = bert_ref.l2_normalize(bert_ref.pool(xmod_ref.xmod_encoder_forward(we, ocfg, ids, mask, device="cuda"),
                                                   mask.cuda(), "mean")).cpu().numpy()
    assert np.abs(got - want).max() < 1e-4
    # a cross-encoder: roberta. + the classification head, one label -> sigmoid
    wc = synthetic_bert_weights(cfg, seed=7, with_head=True, scale=2.0)
    t = {}
    for k, v in wc.items():
        k = "classifier.dense." + k[13:] if k.startswith("pooler.dense.") else \
            "classifier.out_proj." + k[11:] if k.startswith("classifier.") else "roberta." + k
        t[k] = v
    p = _write(tmp_path / "xmod-ce", _conf(cfg), t, tok)
    ce = HuggingFaceCrossEncoder(model_name=p)
    assert ce.colbert is None and ce.activation == "sigmoid"
    pairs = [(texts[0], d) for d in texts[1:]] + [(texts[3], texts[4])]
    got = ce.score(pairs)
    ids, mask = _hf_batch(tok, [a.strip() for a, _ in pairs], [b.strip() for _, b in pairs], ce.max_length)
    with torch.no_grad():
        want = torch.sigmoid(xmod_ref.classifier_head(wc, xmod_ref.xmod_encoder_forward(wc, ocfg, ids, mask,
                                                                                         device="cuda")))[:, 0]
    assert np.abs(got - want.cpu().numpy()).max() < 1e-4


def test_a_missing_language_is_refused_before_any_upload(cuda, tmp_path, monkeypatch):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.tokenizer import load_tokenizer
    cfg, w, lin, _ = synthetic_colbert("tiny-colbert-xm", 1)
    tok = load_tokenizer(None, cfg.vocab_size, xlmr=True)
    p = _write(tmp_path / "colbert-xm", _conf(cfg, architectures=["HF_ColBERT"], default_language=None),
               {**{"roberta." + k: v for k, v in w.items()}, "linear.weight": lin}, tok,
               {"query_maxlen": 16, "doc_maxlen": 64})
    L = _lib()
    n0 = L.launch_count()                          # uploading the weights launches the split-plane kernel
    with pytest.raises(ValueError, match="RMU_XMOD_LANGUAGE"):
        HuggingFaceCrossEncoder(model_name=p)
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "pt_XX")
    with pytest.raises(ValueError, match="language 'pt_XX': it is not one of"):
        HuggingFaceCrossEncoder(model_name=p)
    assert L.launch_count() == n0
    monkeypatch.setenv(W.XMOD_LANGUAGE_ENV, "fr_XX")
    ce = HuggingFaceCrossEncoder(model_name=p)
    assert ce.config.language == "fr_XX" and np.isfinite(ce.score([("a b", "c d e")])).all()
