"""GPU: XLM-RoBERTa / RoBERTa on the encoder, in the regime XLM-R opens: sequences of up to 8192 tokens (the key
super-block loop of E2 runs up to 32 times), position tables of 8194 rows and a 250 002-row word table.  E2 and E3
embed_ln alone against float64 (oracle/encoder_kernels_ref.py, oracle/mpnet_ref.py); the whole stack against the
float64 forward on the split weights (oracle/xlmr_ref.py), with the logits and CLS embeddings bit-identical to the
last hidden state through the debug heads; then the product (HuggingFaceCrossEncoder, HuggingFaceEmbeddings, the vector
store with MMR, ScoredCrossEncoderReranker, the SemanticChunker) against the fp32 oracle.  Bounds follow
tests/test_encoder_kernels_gpu.py and tests/test_encoder_stack_gpu.py (u = 2^-24)."""
import math
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref, chunker_ref, flat_ref
from oracle import encoder_kernels_ref as ref
from oracle import mpnet_ref, xlmr_ref
from ragmeup_b200.documents import Document
from ragmeup_b200.weights import PRESETS, XLMRConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


# ----------------------------------------------------------------------------------------------------- E2, long S
# c_att as in test_encoder_kernels_gpu.py: |err| <= 8 * 2^-22 * max|V| * (1 + A) per sequence and head.  The
# sequences below make the key super-block loop (256 keys at a time) run 3, 4, 8, 17 and 32 times.
C_ATT = 8.0
LONG = [1, 31, 513, 1000, 2048, 4097, 8192]


def _attention(qkv, cu, H, heads):
    T = qkv[0].shape[0]
    ch = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    rc = _lib().lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(_i32(cu)), len(cu) - 1, H, heads,
                                          int(np.diff(cu).max()), 10, _ptr(ch), _ptr(cl), _lib().stream_ptr())
    _lib().check(rc, "rmu_debug_attention")
    torch.cuda.synchronize()
    return ch, cl


@pytest.mark.parametrize("H,heads", [(384, 12), (768, 12)])     # d_h 32 and 64
def test_attention_long_sequences_match_float64(cuda, H, heads):
    rng = np.random.default_rng(H + 8192)
    dh = H // heads
    cu = np.r_[0, np.cumsum(LONG)].astype(np.int64)
    T = int(cu[-1])
    q, k, v = (rng.standard_normal((T, H)) for _ in range(3))
    q *= math.log2(math.e) / math.sqrt(dh)
    qkv = tuple(torch.from_numpy(p).cuda() for p in ref.split_f16(np.concatenate([q, k, v], 1).astype(np.float32)))
    ch, cl = _attention(qkv, cu, H, heads)
    got = ch.double() + cl.double()
    worst = {}
    G = 4                                               # heads per float64 reference call: bounds its S x S memory
    for b, S in enumerate(LONG):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        for h0 in range(0, heads, G):
            cols = torch.cat([torch.arange(part * H + h0 * dh, part * H + (h0 + G) * dh) for part in range(3)]).cuda()
            sub = (qkv[0][t0:t1][:, cols], qkv[1][t0:t1][:, cols])
            want, A = ref.attention_ref(sub[0], sub[1], [0, S], G)
            vv = (sub[0][:, 2 * G * dh:].double() + sub[1][:, 2 * G * dh:].double()).view(S, G, dh)
            bound = 2.0 ** -22 * vv.abs().amax((0, 2))[None, :, None] * (1 + A[:, :, None])
            err = (got[t0:t1, h0 * dh:(h0 + G) * dh] - want).abs().view(S, G, dh)
            worst[S] = max(worst.get(S, 0.0), float((err / bound).max()))
            del want, A
        torch.cuda.empty_cache()
    print(f"\nE2 long H={H} heads={heads}: worst |err|/(2^-22 max|V| (1+A)) by S = "
          + ", ".join(f"{s}: {r:.3g}" for s, r in worst.items()))
    assert max(worst.values()) <= C_ATT, worst


# ------------------------------------------------------------------------------------- E3 embed_ln at XLM-R's tables
C_EMB = 20.0     # test_encoder_kernels_gpu.py's c_emb


def test_embed_ln_positions_at_xlmr_tables(cuda):
    """vocab 250 002, max_pos 8194 (bge-m3), H 1024: positions up to 8193, id 1 mid-sequence in long sequences, ids at
    both ends of the word table"""
    H, V, P = 1024, 250002, 8194
    g = torch.Generator(device="cuda").manual_seed(4)
    word = torch.randn(V, H, device="cuda", generator=g)
    tabs = (word, 0.5 * torch.randn(P, H, device="cuda", generator=g), 0.3 * torch.randn(1, H, device="cuda", generator=g),
            1 + 0.2 * torch.randn(H, device="cuda", generator=g), 0.2 * torch.randn(H, device="cuda", generator=g))
    rng = np.random.default_rng(6)
    seqs = [rng.integers(2, V, n) for n in (8192, 8192, 4097, 513, 3)]
    seqs[0][[0, -1]] = (0, V - 1)                   # no id 1: the last token takes position 8193
    seqs[1][rng.choice(8192, 300, replace=False)] = 1
    seqs[1][[100, 101, 102, 5000]] = 1
    seqs[2][[4000, 4001]] = 1
    lens = [len(s) for s in seqs]
    ids = _i32(np.concatenate(seqs))
    cu = _i32(np.r_[0, np.cumsum(lens)])
    T = ids.numel()
    oh = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    ol = torch.full_like(oh, float("nan"))
    _lib().check(_lib().lib().rmu_debug_embed_ln_pos(_ptr(ids), None, _ptr(cu), len(lens), T, H, V, P, 1, *map(_ptr, tabs),
                                                     1e-5, 1, _ptr(oh), _ptr(ol), _lib().stream_ptr()),
                 "rmu_debug_embed_ln_pos")
    torch.cuda.synchronize()
    got = oh.double() + ol.double()
    want, xhat, sigma, M = mpnet_ref.embed_ln_pos_ref(ids, None, cu, *tabs, 1e-5, pos_mode=1)
    gg, bb = tabs[3].double(), tabs[4].double()
    mag = gg.abs()[None, :] * (1 + xhat.abs()) * (1 + M / sigma) + bb.abs()[None, :]
    split = 2.0 ** -22 * want.abs() + 2.0 ** -25
    ratio = float((((got - want).abs() - split).clamp(min=0) / (U * mag)).max())
    print(f"\nembed_ln at XLM-R tables: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= C_EMB
    p = xlmr_ref.position_ids(torch.from_numpy(seqs[0].astype(np.int64)))
    assert int(p[-1]) == 8193


# -------------------------------------------------------------------------------------------------- whole stack
FLOOR = 4.0
OUTPUTS = ("hidden", "mean", "mean_norm", "cls", "cls_norm", "logits")
# (preset, weight scale, lengths, c, c_mean): c bounds the max and RMS ratios to fp32's error, as in
# test_encoder_stack_gpu.py: twice the worst ratio measured on an H100 (DESIGN.md section 2), rounded up.  c_mean is
# the same rule for the two mean-pooled outputs, whose ratio grows with the sequence length: the fp32 forward's error
# in a mean averages down over the tokens, the device's absolute error does not (mean_norm within 1e-5 at 8192 tokens).
STACK = {
    "bge-reranker-base": ("bge-reranker-base", 1.0, [0, 1, 9, 16, 129, 0, 255, 256, 257, 384, 512, 0], 90, 140),
    "bge-reranker-v2-m3": ("bge-reranker-v2-m3", 1.0, [1, 17, 0, 300, 513, 1100], 80, 150),
    "tiny-xlmr-long x4": ("tiny-xlmr-long", 4.0, [0, 1, 513, 2048, 4097, 8192, 0], 80, 450),
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
    """the fp32 forward one sequence at a time (an 8192-token batch padded to its longest would hold B x S x S
    scores); empty sequences embed as zeros and score the head of a zero CLS row, as the kernels define them"""
    lens = np.diff(cu)
    ocfg = xlmr_ref.XLMRCfg(**asdict(cfg))
    H = cfg.hidden
    out = {k: [] for k in OUTPUTS}
    with torch.no_grad():
        for b, n in enumerate(lens):
            if n == 0:
                z = torch.zeros((1, H), device="cuda")
                for k in ("mean", "mean_norm", "cls", "cls_norm"):
                    out[k].append(z)
                out["logits"].append(xlmr_ref.classifier_head(w32, z[:, None, :]))
                continue
            I = torch.from_numpy(ids[cu[b]:cu[b + 1]].astype(np.int64))[None]
            h = xlmr_ref.xlmr_encoder_forward(w32, ocfg, I, torch.ones_like(I), device="cuda")
            mask = torch.ones_like(I).cuda()
            out["hidden"].append(h[0])
            for mode in ("mean", "cls"):
                e = bert_ref.pool(h, mask, mode)
                out[mode].append(e)
                out[mode + "_norm"].append(bert_ref.l2_normalize(e))
            out["logits"].append(xlmr_ref.classifier_head(w32, h))
    return {k: torch.cat(v).double() for k, v in out.items()}


def _split_heads(enc, w, ids, cu, mx):
    """rmu_encoder_hidden -> rmu_debug_split_planes -> rmu_debug_cls_head / rmu_debug_pool (CLS): the logits and CLS
    embeddings the full stack's heads must equal bit for bit (tests/test_encoder_cls_rows_gpu.py)"""
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


@pytest.mark.parametrize("case", list(STACK))
def test_xlmr_stack_matches_float64_forward(cuda, case):
    from ragmeup_b200.encoder import BertEncoder
    preset, scale, lens, c_rest, c_mean = STACK[case]
    cfg = XLMRConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=19, with_head=True, scale=scale)
    enc = BertEncoder(cfg, w, with_head=True)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    w32 = {k: ref.split_weight(v).float() if k.endswith(ref.GEMM_WEIGHTS) else v for k, v in wd.items()}
    ids, cu, mx = _batch(lens, cfg.vocab_size, 9)
    got = _gpu(enc, ids, cu, mx)
    want = xlmr_ref.xlmr_stack_ref(wd, cfg, ids, cu, "split", device="cuda")
    f32 = _fp32(w32, cfg, ids, cu)
    nonempty = torch.from_numpy(np.diff(cu) > 0).cuda()
    report, fails = [], []
    for name in OUTPUTS:
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
    print(f"\nXLM-R stack {case}:\n  " + "\n  ".join(report))
    for name in ("mean", "cls"):
        assert (got[name][~nonempty] == 0).all()
    assert not fails, f"{case}: beyond {c_rest} (means {c_mean}) x fp32's error: " + "; ".join(fails)
    # the logits and CLS embeddings are the last hidden state's, through the heads alone, bit for bit
    logits, emb = _split_heads(enc, w, ids, cu, mx)
    assert torch.equal(logits, got["logits"]), "logits differ from the heads on rmu_encoder_hidden"
    assert torch.equal(emb[0] + 0.0, got["cls"] + 0.0) and torch.equal(emb[1] + 0.0, got["cls_norm"] + 0.0)
    # host entry points equal the device ones; the longest sequence alone equals its rows in the batch
    assert np.array_equal(enc.classify_host(ids, None, cu), got["logits"].cpu().numpy())
    assert np.array_equal(enc.embed_host(ids, None, cu, "cls", True), got["cls_norm"].cpu().numpy())
    b = int(np.argmax(np.diff(cu)))
    t0, t1 = int(cu[b]), int(cu[b + 1])
    one = _gpu(enc, ids[t0:t1], np.array([0, t1 - t0], np.int32), t1 - t0)
    assert torch.equal(one["hidden"], got["hidden"][t0:t1]) and torch.equal(one["logits"][0], got["logits"][b])
    from ragmeup_b200._lib import RmuError
    n = cfg.max_pos - 1
    with pytest.raises(RmuError, match="max_position_embeddings - 2"):
        enc.embed_tokens(np.full(n, 5, np.int32), None, np.array([0, n], np.int32), n)


# -------------------------------------------------------------------------------------------------------- product
def _copy(tok):
    from tokenizers import Tokenizer
    return Tokenizer.from_str(tok.to_str())


def _texts(tok, n, lo, hi, seed):
    """seeded texts of whole pieces of the synthetic Unigram vocabulary (one or more pieces per word)"""
    words = [p[1:] for p in tok.get_vocab() if p.startswith("▁") and len(p) > 2]
    words.sort()
    rng = np.random.default_rng(seed)
    return [" ".join(words[int(j)] for j in rng.integers(0, len(words), int(rng.integers(lo, hi + 1)))) for _ in range(n)]


@pytest.fixture(scope="module")
def rerankers(cuda):
    from ragmeup_b200.cross_encoder import HuggingFaceCrossEncoder
    from ragmeup_b200.weights import resolve_model
    out = {}
    for scale in (1, 4):
        name = f"synthetic:bge-reranker-base:3:{scale}"
        ce = HuggingFaceCrossEncoder(model_name=name)
        cfg, w, *_ = resolve_model(name, with_head=True)
        out[scale] = (ce, w, xlmr_ref.XLMRCfg(**asdict(cfg)))
    return out


@pytest.mark.parametrize("scale", [1, 4])
@pytest.mark.parametrize("shape", ["ragmeup_14", "bulk_100", "cut_at_max_length"])
def test_score_matches_cross_encoder_predict(rerankers, scale, shape):
    """score() against CrossEncoder.predict restated on the tokenizer's own pair tokenisation (not PairAssembler)"""
    ce, w, ocfg = rerankers[scale]
    assert (ce.max_length, ce.activation, ce.config.num_labels) == (512, "sigmoid", 1)
    n, lo, hi = {"ragmeup_14": (14, 60, 110), "bulk_100": (100, 5, 200), "cut_at_max_length": (12, 520, 900)}[shape]
    query = _texts(ce.tokenizer, 1, 8, 14, seed=scale)[0]
    docs = _texts(ce.tokenizer, n, lo, hi, seed=10 + scale) + (["", "<pad> <mask>"] if shape == "bulk_100" else [])
    pairs = [(query, d) for d in docs]
    if shape == "cut_at_max_length":
        pairs += [(d, query) for d in docs[:3]] + [(docs[3], docs[4])]
    got = ce.score(pairs)
    want = xlmr_ref.cross_encoder_predict(w, ocfg, _copy(ce.tokenizer), pairs, max_length=512, device="cuda")
    ids, _typ, cu = ce._pairs([p[0].strip() for p in pairs], [p[1].strip() for p in pairs])
    raw = ce.client.classify_host(ids, None, cu)
    want_raw = xlmr_ref.cross_encoder_predict(w, ocfg, _copy(ce.tokenizer), pairs, max_length=512, activation="identity",
                                              device="cuda")
    if shape == "cut_at_max_length":
        assert (np.diff(cu) == 512).all()
    assert got.shape == (len(pairs),) and got.dtype == np.float32
    scale_raw = max(1.0, float(np.abs(want_raw).max()))
    assert np.abs(raw[:, 0] - want_raw).max() < 2e-3 * scale_raw, np.abs(raw[:, 0] - want_raw).max()
    assert np.abs(got - want).max() < 1e-3
    t = ce.score_tensor(pairs).cpu().numpy()
    assert np.abs(t - got).max() < 1e-6


def test_pairs_match_pair_tokenisation(rerankers):
    from ragmeup_b200.tokenizer import RaggedTokenizer
    ce = rerankers[1][0]
    docs = _texts(ce.tokenizer, 30, 1, 700, seed=5)
    a, b = [docs[0]] * 30, docs
    got, want = ce._pairs(a, b), RaggedTokenizer(ce.tokenizer, 512)(a, b)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))


@pytest.fixture(scope="module")
def embedders(cuda):
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.weights import resolve_model
    out = {}
    for name in ("multilingual-e5-small", "bge-m3", "paraphrase-multilingual-mpnet-base-v2"):
        emb = HuggingFaceEmbeddings(model_name=f"synthetic:{name}:3")
        cfg, w, *_ = resolve_model(emb.model_name, with_head=False)
        out[name] = (emb, w, xlmr_ref.XLMRCfg(**asdict(cfg)))
    return out


@pytest.mark.parametrize("name,pooling,normalize,max_len,long", [
    ("multilingual-e5-small", "mean", True, 512, 700),
    ("bge-m3", "cls", True, 8192, 1500),                       # texts past 512 tokens
    ("paraphrase-multilingual-mpnet-base-v2", "mean", False, 128, 300),
])
def test_embed_documents_and_query_match_oracle(embedders, name, pooling, normalize, max_len, long):
    emb, w, ocfg = embedders[name]
    assert (emb.pooling, emb.normalize, emb.max_seq_length) == (pooling, normalize, max_len)
    texts = _texts(emb.tokenizer, 20, 3, long, 11) + ["a <pad> in the text", "<pad>", "line one\nline two  ", ""]
    lens = np.diff(emb._ragged(texts)[2])
    if name == "bge-m3":
        assert lens.max() > 1024
    got = np.asarray(emb.embed_documents(texts), np.float32)
    want = np.asarray(xlmr_ref.hf_embed_documents(w, ocfg, _copy(emb.tokenizer), texts, pooling=pooling,
                                                  normalize=normalize, max_seq_length=max_len, device="cuda"), np.float32)
    assert got.shape == (len(texts), ocfg.hidden)
    assert np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))
    assert np.array_equal(np.asarray(emb.embed_query(texts[0]), np.float32), got[0])


def test_chunking_at_max_tokens_per_call(cuda):
    """T = MAX_TOKENS_PER_CALL + 1 through encode_tensor and embed_host: two chunks, every checked row bit-identical
    to the text alone"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL, BertEncoder
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny-xlmr")
    vocab = sorted(p[1:] for p in emb.tokenizer.get_vocab() if p.startswith("▁") and len(p) > 2)
    words = [w for w, e in zip(vocab, emb.tokenizer.encode_batch(vocab, add_special_tokens=False)) if len(e.ids) == 1]
    rng = np.random.default_rng(1)
    n = MAX_TOKENS_PER_CALL // 64
    texts = [" ".join(rng.choice(words, c)) for c in [62] * (n - 1) + [61, 0]]
    ids, typ, cu = emb._ragged(texts)
    assert int(cu[-1]) == MAX_TOKENS_PER_CALL + 1 and len(list(BertEncoder._chunks(cu, MAX_TOKENS_PER_CALL))) == 2
    out = emb.encode_tensor(texts)
    host = emb.client.embed_host(ids, None, cu, emb.pooling, emb.normalize)
    for i in sorted({0, n // 2, n - 2, n - 1, len(texts) - 1}):
        alone = emb.encode_tensor([texts[i]])[0]
        assert torch.equal(out[i], alone) and torch.equal(torch.from_numpy(host[i]), alone.cpu()), i


def test_mmr_then_xlmr_rerank_and_chunker(embedders, rerankers):
    """Milvus MMR on an XLM-R embedder, then ScoredCrossEncoderReranker with the XLM-R reranker; the SemanticChunker on
    the XLM-R embedder"""
    from ragmeup_b200.chunker import SemanticChunker
    from ragmeup_b200.reranker import ScoredCrossEncoderReranker
    from ragmeup_b200.vectorstore import Milvus
    emb, w, ocfg = embedders["multilingual-e5-small"]
    ce, cw, ccfg = rerankers[1]
    docs = _texts(emb.tokenizer, 300, 40, 90, 21)
    queries = _texts(emb.tokenizer, 3, 5, 20, 22)
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="xlmr")
    db.add_documents([Document(t, {"id": f"id{i}"}) for i, t in enumerate(docs)], ids=[f"id{i}" for i in range(300)])
    X = xlmr_ref.st_encode(w, ocfg, _copy(emb.tokenizer), docs, "mean", True, 512, device="cuda")
    retriever = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    rr = ScoredCrossEncoderReranker(model=ce, top_n=3)
    for qtext in queries:
        qv = np.asarray(xlmr_ref.hf_embed_documents(w, ocfg, _copy(emb.tokenizer), [qtext], device="cuda")[0], np.float32)
        want = flat_ref.mmr_search(qv[None], X, 10, "l2", fetch_k=20, lambda_mult=0.5)[0]
        found = retriever.invoke(qtext)
        assert [d.metadata["pk"] for d in found] == [f"id{r}" for r in want]
        top = rr.compress_documents(found, qtext)
        pairs = [(qtext, d.page_content) for d in found]
        got = ce.score(pairs)
        order = sorted(range(len(found)), key=lambda i: got[i], reverse=True)[:3]
        assert [d.page_content for d in top] == [found[i].page_content for i in order]
        assert [d.metadata["relevance_score"] for d in top] == [got[i] for i in order]
        s = xlmr_ref.cross_encoder_predict(cw, ccfg, _copy(ce.tokenizer), pairs, device="cuda")
        assert np.abs(got - s).max() < 1e-3
    text = " ".join(t + "." for t in _texts(emb.tokenizer, 40, 6, 14, 23))
    sc = SemanticChunker(emb, breakpoint_threshold_type="percentile")
    got = sc.split_text(text)
    want, _ = chunker_ref.split_text(text, emb.embed_documents, kind="percentile", amount=None, number_of_chunks=None)
    assert got == want and " ".join(got) == text and len(got) >= 2
