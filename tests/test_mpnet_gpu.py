"""GPU: MPNet on the encoder.  E2 with the relative position bias and E3 embed_ln with the padding-offset positions,
each alone against the float64 references of oracle/mpnet_ref.py; the whole stack against the float64 forward on the
split weights; then the product (HuggingFaceEmbeddings, the vector store with MMR, the SemanticChunker) against the fp32
oracle.  Bounds follow tests/test_encoder_kernels_gpu.py and tests/test_encoder_stack_gpu.py (u = 2^-24)."""
import math
from dataclasses import asdict

import numpy as np
import pytest
import torch

from oracle import bert_ref, chunker_ref, flat_ref
from oracle import encoder_kernels_ref as ref
from oracle import mpnet_ref
from ragmeup_b200.documents import Document
from ragmeup_b200.weights import PRESETS, MPNetConfig, synthetic_bert_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _lib():
    from ragmeup_b200 import _lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _table(bias):
    """[32, heads] fp32 -> the [heads, 255] device table rmu_encoder_create builds"""
    heads = bias.shape[1]
    tab = np.zeros((heads, 255), np.float32)
    _lib().check(_lib().lib().rmu_relative_bias_table(np.ascontiguousarray(bias, np.float32).ctypes.data, 32, heads,
                                                      tab.ctypes.data), "rmu_relative_bias_table")
    return torch.from_numpy(tab).cuda()


# ----------------------------------------------------------------------------------------------------- E2 + bias
# c_att as in test_encoder_kernels_gpu.py, in units of 2^-22 max|V| (1 + A), with A now max over the row's keys of
# sum_d |q_d k_d| + |bias|: the bias entry is bias * log2(e) rounded to fp32 (u |bias|) and one more fp32 add after
# the QK sum (u (|qk| + |bias|)), so the score error is still a few u * A and each p = 2^s moves by ln2 times that;
# the P split, ex2.approx and the P V accumulation are unchanged.  c = 8.  A bias read at i - j, or left in natural
# units, moves scores by O(|bias|) ~ 1, millions of times the bound.
C_ATT = 8.0
EDGES = [1, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 160, 161, 255, 256, 257, 300, 512]


def _attention(qkv, cu, H, heads, tab, cls_q=None):
    T = qkv[0].shape[0]
    rows = T if cls_q is None else len(cu) - 1
    ch = torch.full((rows, H), float("nan"), dtype=torch.float16, device="cuda")
    cl = torch.full_like(ch, float("nan"))
    cu_d = _i32(cu)
    rc = _lib().lib().rmu_debug_attention_bias(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(None if cls_q is None else cls_q[0]),
                                               _ptr(None if cls_q is None else cls_q[1]), _ptr(cu_d), len(cu) - 1, H,
                                               heads, int(np.diff(cu).max()), _ptr(tab), _ptr(ch), _ptr(cl),
                                               _lib().stream_ptr())
    _lib().check(rc, "rmu_debug_attention_bias")
    torch.cuda.synchronize()
    return ch, cl


def _qkv(rng, lens, H, heads):
    dh = H // heads
    cu = np.r_[0, np.cumsum(lens)].astype(np.int64)
    T = int(cu[-1])
    q, k, v = (rng.standard_normal((T, H)) for _ in range(3))
    q *= math.log2(math.e) / math.sqrt(dh)
    return tuple(torch.from_numpy(p).cuda() for p in ref.split_f16(np.concatenate([q, k, v], 1).astype(np.float32))), cu


@pytest.mark.parametrize("H,heads", [(384, 12), (768, 12)])          # d_h 32 and 64
def test_biased_attention_matches_float64(cuda, H, heads):
    rng = np.random.default_rng(H + heads)
    qkv, cu = _qkv(rng, EDGES, H, heads)
    bias = (2.0 * rng.standard_normal((32, heads))).astype(np.float32)   # asymmetric: i - j differs from j - i
    tab = _table(bias)
    ch, cl = _attention(qkv, cu, H, heads, tab)
    got = ch.double() + cl.double()
    want, A = mpnet_ref.attention_bias_ref(qkv[0], qkv[1], cu, heads, tab)
    dh = H // heads
    v = qkv[0][:, 2 * H:].double() + qkv[1][:, 2 * H:].double()
    worst = 0.0
    for b in range(len(EDGES)):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        vmax = v[t0:t1].abs().view(t1 - t0, heads, dh).amax((0, 2))
        bound = 2.0 ** -22 * vmax[None, :, None] * (1 + A[t0:t1, :, None])
        worst = max(worst, float(((got[t0:t1] - want[t0:t1]).abs().view(t1 - t0, heads, dh) / bound).max()))
    print(f"\nE2+bias H={H} heads={heads}: worst |err|/(2^-22 max|V| (1+A)) = {worst:.3g}")
    assert worst <= C_ATT, f"E2 with bias: error {worst:.3g} exceeds {C_ATT}"
    # CLS mode: query row 0 of each sequence from compact Q planes, bit-identical to row 0 of the full kernel
    starts = torch.from_numpy(cu[:-1]).cuda()
    cls_q = (qkv[0][starts, :H].contiguous(), qkv[1][starts, :H].contiguous())
    kh, kl = _attention(qkv, cu, H, heads, tab, cls_q)
    assert _bits_equal(kh, ch[starts]) and _bits_equal(kl, cl[starts]), "CLS mode differs from row 0 of the full kernel"
    # an all-zero table: bit-identical to the kernel without the bias
    zh, zl = _attention(qkv, cu, H, heads, torch.zeros_like(tab))
    bh = torch.full_like(zh, float("nan")); bl = torch.full_like(zl, float("nan"))
    _lib().check(_lib().lib().rmu_debug_attention(_ptr(qkv[0]), _ptr(qkv[1]), _ptr(_i32(cu)), len(cu) - 1, H, heads,
                                                  int(np.diff(cu).max()), 10, _ptr(bh), _ptr(bl), _lib().stream_ptr()),
                 "rmu_debug_attention")
    torch.cuda.synchronize()
    assert _bits_equal(zh, bh) and _bits_equal(zl, bl), "a zero bias table changes the result"


# ----------------------------------------------------------------------------------------- E3 embed_ln + positions
C_EMB = 20.0     # test_encoder_kernels_gpu.py's c_emb: the position rule picks a row, it adds no arithmetic


def _embed(ids, cu, tabs, mode, eps=1e-5):
    word, pos, typ, g, b = tabs
    T, H = ids.numel(), word.shape[1]
    oh = torch.full((T, H), float("nan"), dtype=torch.float16, device="cuda")
    ol = torch.full_like(oh, float("nan"))
    rc = _lib().lib().rmu_debug_embed_ln_pos(_ptr(ids), None, _ptr(cu), cu.numel() - 1, T, H, word.shape[0], pos.shape[0],
                                             typ.shape[0], _ptr(word), _ptr(pos), _ptr(typ), _ptr(g), _ptr(b), eps, mode,
                                             _ptr(oh), _ptr(ol), _lib().stream_ptr())
    _lib().check(rc, "rmu_debug_embed_ln_pos")
    torch.cuda.synchronize()
    return oh, ol


def test_embed_ln_positions_match_float64(cuda):
    """id 1 in the middle of sequences (also several in a row and past the first 32 tokens), at the start, as the whole
    sequence; sequences long enough that the ballot loop runs 16 rounds; positions past max_pos clamp"""
    H, V, P = 768, 2000, 514
    g = torch.Generator(device="cuda").manual_seed(3)
    tabs = (torch.randn(V, H, device="cuda", generator=g), 0.5 * torch.randn(P, H, device="cuda", generator=g),
            torch.zeros(1, H, device="cuda"), 1 + 0.2 * torch.randn(H, device="cuda", generator=g),
            0.2 * torch.randn(H, device="cuda", generator=g))
    rng = np.random.default_rng(5)
    seqs = []
    for n in (1, 5, 33, 100, 512, 40, 7, 600):
        s = rng.integers(2, V, n)
        seqs.append(s)
    seqs[1][2] = 1                                  # mid-sequence
    seqs[2][[0, 31, 32]] = 1                        # at the start and across the first ballot round
    seqs[3][[10, 11, 12, 70]] = 1
    seqs[4][rng.choice(512, 40, replace=False)] = 1
    seqs[5][:] = 1                                  # the whole sequence
    seqs[6][0] = 1
    lens = [len(s) for s in seqs]
    ids = _i32(np.concatenate(seqs))
    cu = _i32(np.r_[0, np.cumsum(lens)])
    oh, ol = _embed(ids, cu, tabs, 1)
    got = oh.double() + ol.double()
    want, xhat, sigma, M = mpnet_ref.embed_ln_pos_ref(ids, None, cu, *tabs, 1e-5, pos_mode=1)
    gg, bb = tabs[3].double(), tabs[4].double()
    mag = gg.abs()[None, :] * (1 + xhat.abs()) * (1 + M / sigma) + bb.abs()[None, :]
    split = 2.0 ** -22 * want.abs() + 2.0 ** -25
    ratio = float((((got - want).abs() - split).clamp(min=0) / (U * mag)).max())
    print(f"\nembed_ln positions: worst |err|/(u*mag) = {ratio:.3g}")
    assert ratio <= C_EMB
    # every token of the all-id-1 sequence takes position 1: all its rows are the same
    t0 = sum(lens[:5])
    assert _bits_equal(oh[t0:t0 + 40], oh[t0:t0 + 1].expand(40, H))
    # mode 0 is rmu_debug_embed_ln, bit for bit
    zh, zl = _embed(ids, cu, tabs, 0)
    word, pos, typ, gm, bt = tabs
    rh = torch.full_like(zh, float("nan")); rl = torch.full_like(zl, float("nan"))
    _lib().check(_lib().lib().rmu_debug_embed_ln(_ptr(ids), None, _ptr(cu), cu.numel() - 1, ids.numel(), H, V, P, 1,
                                                 _ptr(word), _ptr(pos), _ptr(typ), _ptr(gm), _ptr(bt), 1e-5, _ptr(rh),
                                                 _ptr(rl), _lib().stream_ptr()), "rmu_debug_embed_ln")
    torch.cuda.synchronize()
    assert _bits_equal(zh, rh) and _bits_equal(zl, rl)


# -------------------------------------------------------------------------------------------------- whole stack
FLOOR = 4.0
OUTPUTS = ("hidden", "mean", "mean_norm", "cls", "cls_norm")
LENS = [0, 1, 9, 16, 129, 0, 255, 256, 257, 384, 512, 0]
# (preset, weight scale, lengths, c): c bounds the max and RMS ratios to fp32's error, as in test_encoder_stack_gpu.py:
# twice the worst ratio over the five outputs measured on an H100 (DESIGN.md section 2), rounded up
STACK = {
    "all-mpnet-base-v2": ("all-mpnet-base-v2", 1.0, LENS, 48),
    "tiny-mpnet x4": ("tiny-mpnet", 4.0, [0, 1, 2, 64, 127, 128, 0, 33], 10),
}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


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
    out = {"hidden": enc.hidden_tokens(ids, None, cu, mx)}
    for mode in ("mean", "cls"):
        out[mode] = enc.embed_tokens(ids, None, cu, mx, mode, False)
        out[mode + "_norm"] = enc.embed_tokens(ids, None, cu, mx, mode, True)
    torch.cuda.synchronize()
    return out


def _fp32(w32, cfg, ids, cu):
    lens = np.diff(cu)
    S = int(lens.max())
    I = np.ones((len(lens), S), np.int64); M = np.zeros_like(I)
    for b, n in enumerate(lens):
        I[b, :n] = ids[cu[b]:cu[b + 1]]
        M[b, :n] = 1
    with torch.no_grad():
        h = mpnet_ref.mpnet_encoder_forward(w32, mpnet_ref.MPNetCfg(**asdict(cfg)), torch.from_numpy(I),
                                            torch.from_numpy(M), device="cuda")
        mask = torch.from_numpy(M).cuda()
        out = {"hidden": torch.cat([h[b, :n] for b, n in enumerate(lens)])}
        for mode in ("mean", "cls"):
            out[mode] = bert_ref.pool(h, mask, mode)
            out[mode + "_norm"] = bert_ref.l2_normalize(out[mode])
    return {k: v.double() for k, v in out.items()}


@pytest.mark.parametrize("case", list(STACK))
def test_mpnet_stack_matches_float64_forward(cuda, case):
    from ragmeup_b200.encoder import BertEncoder
    preset, scale, lens, c = STACK[case]
    cfg = MPNetConfig(**asdict(PRESETS[preset][0]))
    w = synthetic_bert_weights(cfg, seed=17, with_head=False, scale=scale)
    enc = BertEncoder(cfg, w, with_head=False)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    w32 = {k: ref.split_weight(v).float() if k.endswith(ref.GEMM_WEIGHTS) else v for k, v in wd.items()}
    ids, cu, mx = _batch(lens, cfg.vocab_size, 9)
    got = _gpu(enc, ids, cu, mx)
    want = mpnet_ref.mpnet_stack_ref(wd, cfg, ids, cu, "split", device="cuda")
    f32 = _fp32(w32, cfg, ids, cu)
    nonempty = torch.from_numpy(np.diff(cu) > 0).cuda()
    report, fails = [], []
    for name in OUTPUTS:
        g, w_, f = got[name].double(), want[name], f32[name]
        assert torch.isfinite(g).all(), name
        rows = slice(None) if name == "hidden" else nonempty
        d = (g - w_).abs(); e = (f[rows] - w_[rows]).abs()
        gmax, grms, fmax, frms = float(d.max()), float(d.pow(2).mean().sqrt()), float(e.max()), float(e.pow(2).mean().sqrt())
        mag_max, mag_rms = float(w_.abs().max()), float(w_.pow(2).mean().sqrt())
        report.append(f"{name} max {gmax:.3g} / fp32 {fmax:.3g} = {gmax / fmax:.3g}, rms {grms:.3g} / {frms:.3g} = "
                      f"{grms / frms:.3g}")
        if gmax > c * fmax + FLOOR * U * mag_max or grms > c * frms + FLOOR * U * mag_rms:
            fails.append(report[-1])
    print(f"\nMPNet stack {case}:\n  " + "\n  ".join(report))
    for name in ("mean", "cls"):
        assert (got[name][~nonempty] == 0).all()
    assert not fails, f"{case}: beyond {c} x fp32's error: " + "; ".join(fails)
    # each sequence alone equals its rows in the batch; one token past max_pos - 2 is refused
    for b in (int(np.argmax(np.diff(cu))), 2):
        t0, t1 = int(cu[b]), int(cu[b + 1])
        one = _gpu(enc, ids[t0:t1], np.array([0, t1 - t0], np.int32), t1 - t0)
        assert torch.equal(one["hidden"], got["hidden"][t0:t1]) and torch.equal(one["cls"][0], got["cls"][b])
    from ragmeup_b200._lib import RmuError
    n = cfg.max_pos - 1
    with pytest.raises(RmuError, match="max_position_embeddings - 2"):
        enc.embed_tokens(np.full(n, 5, np.int32), None, np.array([0, n], np.int32), n)


# -------------------------------------------------------------------------------------------------------- product
@pytest.fixture(scope="module")
def mpnet_models(cuda):
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.weights import resolve_model
    out = {}
    for name in ("all-mpnet-base-v2", "multi-qa-mpnet-base-dot-v1"):
        emb = HuggingFaceEmbeddings(model_name=f"synthetic:{name}:3")
        cfg, w, *_ = resolve_model(emb.model_name, with_head=False)
        out[name] = (emb, w, mpnet_ref.MPNetCfg(**asdict(cfg)))
    return out


def _texts(n, lo, hi, seed):
    from ragmeup_b200.tokenizer import synthetic_mpnet_vocab, synthetic_sentences
    return synthetic_sentences(synthetic_mpnet_vocab(30527), n, lo, hi, seed=seed)


@pytest.mark.parametrize("name", ["all-mpnet-base-v2", "multi-qa-mpnet-base-dot-v1"])
def test_embed_documents_and_query_match_oracle(mpnet_models, name):
    emb, w, ocfg = mpnet_models[name]
    pooling, normalize = {"all-mpnet-base-v2": ("mean", True), "multi-qa-mpnet-base-dot-v1": ("cls", False)}[name]
    assert (emb.pooling, emb.normalize, emb.max_seq_length) == (pooling, normalize, PRESETS[name][2])
    texts = _texts(30, 3, 400, 11) + ["a <pad> in the text", "<pad>", "line one\nline two  ", ""]
    got = np.asarray(emb.embed_documents(texts), np.float32)
    want = np.asarray(mpnet_ref.hf_embed_documents(w, ocfg, emb.tokenizer, texts, pooling=pooling, normalize=normalize,
                                                   max_seq_length=emb.max_seq_length), np.float32)
    assert got.shape == (len(texts), 768)
    assert np.abs(got - want).max() < 1e-3 * max(1.0, float(np.abs(want).max()))
    q = np.asarray(emb.embed_query(texts[0]))
    assert np.array_equal(q, got[0])


def test_chunking_at_max_tokens_per_call(cuda):
    """T = MAX_TOKENS_PER_CALL + 1 through encode_tensor and embed_host: two chunks, every checked row bit-identical
    to the text alone"""
    from ragmeup_b200.embeddings import HuggingFaceEmbeddings
    from ragmeup_b200.encoder import MAX_TOKENS_PER_CALL, BertEncoder
    emb = HuggingFaceEmbeddings(model_name="synthetic:tiny-mpnet")
    vocab = [w for w in emb.tokenizer.get_vocab() if w.isalpha() and len(w) > 1][:300]
    words = [w for w, e in zip(vocab, emb.tokenizer.encode_batch(vocab, add_special_tokens=False)) if len(e.ids) == 1]
    rng = np.random.default_rng(1)
    n = MAX_TOKENS_PER_CALL // 64
    texts = [" ".join(rng.choice(words, c)) for c in [62] * (n - 1) + [61, 0]]
    ids, typ, cu = emb._ragged(texts)
    assert int(cu[-1]) == MAX_TOKENS_PER_CALL + 1 and len(list(BertEncoder._chunks(cu, MAX_TOKENS_PER_CALL))) == 2
    out = emb.encode_tensor(texts)
    host = emb.client.embed_host(ids, typ, cu, emb.pooling, emb.normalize)
    for i in sorted({0, n // 2, n - 2, n - 1, len(texts) - 1}):
        alone = emb.encode_tensor([texts[i]])[0]
        assert torch.equal(out[i], alone) and torch.equal(torch.from_numpy(host[i]), alone.cpu()), i


def test_vector_store_mmr_and_chunker_on_mpnet(mpnet_models):
    from ragmeup_b200.chunker import SemanticChunker
    from ragmeup_b200.vectorstore import Milvus
    emb, w, ocfg = mpnet_models["all-mpnet-base-v2"]
    docs = _texts(300, 40, 90, 21)
    queries = _texts(4, 5, 20, 22)
    db = Milvus.from_documents([], emb, drop_old=True, connection_args={"uri": "data.db"}, collection_name="mp")
    db.add_documents([Document(t, {"id": f"id{i}"}) for i, t in enumerate(docs)], ids=[f"id{i}" for i in range(300)])
    X = mpnet_ref.st_encode(w, ocfg, emb.tokenizer, docs, "mean", True, emb.max_seq_length)
    retriever = db.as_retriever(search_type="mmr", search_kwargs={"k": 10})
    for qtext in queries:
        qv = np.asarray(mpnet_ref.hf_embed_documents(w, ocfg, emb.tokenizer, [qtext], max_seq_length=384)[0], np.float32)
        want = flat_ref.mmr_search(qv[None], X, 10, "l2", fetch_k=20, lambda_mult=0.5)[0]
        assert [d.metadata["pk"] for d in retriever.invoke(qtext)] == [f"id{r}" for r in want]
    text = " ".join(s + "." for s in _texts(40, 6, 14, 23))
    sc = SemanticChunker(emb, breakpoint_threshold_type="percentile")
    got = sc.split_text(text)
    want, _ = chunker_ref.split_text(text, emb.embed_documents, kind="percentile", amount=None, number_of_chunks=None)
    assert got == want and " ".join(got) == text and len(got) >= 2
